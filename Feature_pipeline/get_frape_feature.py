#!/usr/bin/env python
"""Drop-in for deep_ctr/Feature_pipeline/get_frape_feature.py on the H100: same flags (:32-51), same outputs (each
<input_dir>/*libsvm -> path.split('.')[0] + '_.libsvm' with the label -1 rewritten to 0, byte for byte), computed on
the GPU.  As in the reference, --output_dir is echoed and otherwise ignored.  e.g.
  python Feature_pipeline/get_frape_feature.py --input_dir=./data/frappe"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main(argv=None):
    parser = argparse.ArgumentParser()
    parser.add_argument("--threads", type=int, default=10, help="threads num (accepted, unused: the GPU does the work)")
    parser.add_argument("--input_dir", type=str, default="", help="input data dir")
    parser.add_argument("--output_dir", type=str, default="", help="feature map output dir (unused, as in the reference)")
    FLAGS, _ = parser.parse_known_args(argv)
    print("threads ", FLAGS.threads)
    print("input_dir ", FLAGS.input_dir)
    print("output_dir ", FLAGS.output_dir)

    from tf_repos_b200.smart_feature import frappe_feature, frappe_outputs
    print("file_list size ", len(frappe_outputs(FLAGS.input_dir)))
    return frappe_feature(FLAGS.input_dir)


if __name__ == "__main__":
    main()
