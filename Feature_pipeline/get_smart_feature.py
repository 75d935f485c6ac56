#!/usr/bin/env python
"""Drop-in for deep_ctr/Feature_pipeline/get_smart_feature.py on the H100: same flags (:92-117), same outputs
(tr_<piece>.libsvm per input, or va.libsvm / te.libsvm, byte for byte), computed on the GPU.  e.g.
  python Feature_pipeline/get_smart_feature.py --input_dir=./data/smart --output_dir=./data/smart/ --task_type=tr
--build_feature_map (not in the reference) first builds output_dir + 'feature_map' from the tr inputs with the
reference's get_feature_map, whose call the reference leaves commented out.  The last line printed is the
--field_size / --feature_size to pass to Model_pipeline/*.py."""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _bool(v):
    return str(v).lower() in ("1", "true", "yes", "y")


def main(argv=None):
    parser = argparse.ArgumentParser()
    parser.add_argument("--threads", type=int, default=10, help="threads num (accepted, unused: the GPU does the work)")
    parser.add_argument("--input_dir", type=str, default="", help="input data dir")
    parser.add_argument("--output_dir", type=str, default="", help="feature map output dir")
    parser.add_argument("--task_type", type=str, default="tr", help="{tr,va,te}")
    parser.add_argument("--build_feature_map", type=_bool, default=False,
                        help="build output_dir + 'feature_map' from the tr inputs first")
    FLAGS, _ = parser.parse_known_args(argv)
    print("threads ", FLAGS.threads)
    print("input_dir ", FLAGS.input_dir)
    print("output_dir ", FLAGS.output_dir)
    print("task_type ", FLAGS.task_type)

    from tf_repos_b200.smart_feature import input_files, smart_feature
    print("file_list size ", len(input_files(FLAGS.input_dir, FLAGS.task_type)))
    out = smart_feature(FLAGS.input_dir, FLAGS.output_dir, FLAGS.task_type,
                        build_feature_map_first=FLAGS.build_feature_map)
    fids = [t[1] for t in (line.split() for line in open(FLAGS.output_dir + "feature_map", "rb")) if len(t) > 1]
    size = max([int(f) for f in fids if f.isdigit()], default=0) + 1
    print(f"feature_size {size}  (train with --field_size=126 --feature_size={size})")
    return out


if __name__ == "__main__":
    main()
