#!/usr/bin/env python
"""Drop-in for deep_ctr/Feature_pipeline/get_aliccp_tfrecord.py (and DeepMTL/Feature_pipeline/get_tfrecord.py,
get_ai_tfrecord.py) on the H100: same flags (:25-27), same glob, naming and mkdir (:39-40, :104-107); every
input_dir/*-* file becomes output_dir/<basename>.tfrecord, computed on the GPU.  e.g.
  python Feature_pipeline/get_aliccp_tfrecord.py --input_dir=./data/aliccp/ --output_dir=./data/aliccp/tfrecord/
The last line printed is the --field_size to pass to Model_pipeline/DIN.py and DeepCvrMTL.py."""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main(argv=None):
    parser = argparse.ArgumentParser()
    parser.add_argument("--input_dir", type=str, default="./", help="input dir")
    parser.add_argument("--output_dir", type=str, default="./", help="output dir")
    parser.add_argument("--threads", type=int, default=16, help="threads num (accepted, unused: the GPU does the work)")
    FLAGS, _ = parser.parse_known_args(argv)

    from tf_repos_b200.aliccp_tfrecord import convert
    out = convert(FLAGS.input_dir, FLAGS.output_dir)
    print("total files: %d" % len(out["files"]))
    print("field_size 11  (train with --field_size=11)")
    return out


if __name__ == "__main__":
    main()
