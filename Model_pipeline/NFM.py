#!/usr/bin/env python
"""Drop-in for deep_ctr/Model_pipeline/NFM.py on the H100 engine (same flags and per-model defaults)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tf_repos_b200 import flags  # noqa: E402
from tf_repos_b200.flags import FLAGS  # noqa: E402

flags.define_common(embedding_size=64, batch_size=128, learning_rate=0.05, l2_reg=0.001, deep_layers="128,64",
                    dropout="0.5,0.8,0.8")      # NFM.py:40-54

def main():
    FLAGS._parse()
    from tf_repos_b200.nfm import NFM
    from tf_repos_b200.estimator import run
    run(lambda: NFM(FLAGS.field_size, FLAGS.feature_size, FLAGS.embedding_size, FLAGS.batch_size,
                    deep_layers=FLAGS.deep_layers, dropout=FLAGS.dropout, l2_reg=FLAGS.l2_reg,
                    learning_rate=FLAGS.learning_rate, optimizer=FLAGS.optimizer, update_mode=FLAGS.update_mode,
                 batch_norm=FLAGS.batch_norm, batch_norm_decay=FLAGS.batch_norm_decay), "NFM")


if __name__ == "__main__":
    main()
