#!/usr/bin/env python
"""Drop-in for DeepMTL/Feature_pipeline's join, stat and remap jobs (get_join_sample.sh, get_stat_feat.sh,
get_remap_fid.sh) on the H100: every file of input_dir/tr/ and input_dir/te/ (e.g. sample_skeleton_train.csv and
common_features_train.csv in tr/, the test pair in te/) becomes output_dir/tr/part-%05d, output_dir/te/part-%05d and
output_dir/feat_cnts, computed on the GPU.  e.g.
  python Feature_pipeline/get_aliccp_sample.py --input_dir=./data/aliccp/raw/ --output_dir=./data/aliccp/sample/
  python Feature_pipeline/get_aliccp_tfrecord.py --input_dir=./data/aliccp/sample/tr --output_dir=./data/aliccp/tr
The last line printed is the --feature_size to pass to Model_pipeline/DeepCvrMTL.py and DIN.py."""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main(argv=None):
    parser = argparse.ArgumentParser()
    parser.add_argument("--input_dir", type=str, default="./", help="input dir (holds tr/ and te/)")
    parser.add_argument("--output_dir", type=str, default="./", help="output dir")
    parser.add_argument("--cutoff", type=int, default=20, help="keep fids seen at least this many times in tr")
    parser.add_argument("--parts", type=int, default=100, help="part files per set (the join job's reducers)")
    parser.add_argument("--seed", type=int, default=0, help="seed of the shuffle key")
    FLAGS, _ = parser.parse_known_args(argv)

    from tf_repos_b200.aliccp_sample import prepare
    out = prepare(FLAGS.input_dir, FLAGS.output_dir, cutoff=FLAGS.cutoff, parts=FLAGS.parts, seed=FLAGS.seed)
    for name in ("tr", "te"):
        s = out[name]
        print("%s: %d lines, %d samples (%d without a common record), %d common records (%d superseded), "
              "%d y=0/z=1 filtered, %d skipped, %d with an empty feature field"
              % (name, s["lines"], s["samples"], s["no_common"], s["commons"], s["commons_superseded"], s["filtered"],
                 s["malformed"], s["empty_lines"]))
    print("kept fids: %d" % out["kept_fids"])
    print("feature_size %d  (train with --feature_size=%d)" % (out["feature_size"], out["feature_size"]))
    return out


if __name__ == "__main__":
    main()
