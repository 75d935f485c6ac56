#!/usr/bin/env python
"""Drop-in for deep_ctr/Feature_pipeline/get_criteo_feature.py on the H100: same flags (:171-197), same outputs
(tr.libsvm, va.libsvm, te.libsvm byte for byte; feature_map as a set of lines), computed on the GPU.  e.g.
  python Feature_pipeline/get_criteo_feature.py --input_dir=./data/criteo/ --output_dir=./data/criteo/ --cutoff=200
The last line printed is the --feature_size to pass to Model_pipeline/*.py (with --field_size=39)."""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main(argv=None):
    parser = argparse.ArgumentParser()
    parser.add_argument("--threads", type=int, default=2, help="threads num (accepted, unused: the GPU does the work)")
    parser.add_argument("--input_dir", type=str, default="", help="input data dir")
    parser.add_argument("--output_dir", type=str, default="", help="feature map output dir")
    parser.add_argument("--cutoff", type=int, default=200, help="cutoff long-tailed categorical values")
    FLAGS, _ = parser.parse_known_args(argv)
    print("threads ", FLAGS.threads)
    print("input_dir ", FLAGS.input_dir)
    print("output_dir ", FLAGS.output_dir)
    print("cutoff ", FLAGS.cutoff)

    from tf_repos_b200.criteo_feature import preprocess
    out = preprocess(FLAGS.input_dir, FLAGS.output_dir, cutoff=FLAGS.cutoff)
    print(f"feature_size {out['feature_size']}  (train with --field_size=39 --feature_size={out['feature_size']})")
    return out


if __name__ == "__main__":
    main()
