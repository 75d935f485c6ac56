#!/usr/bin/env python
"""Drop-in for deep_ctr/Model_pipeline/AFM.py on the H100 engine (same flags and per-model defaults)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tf_repos_b200 import flags  # noqa: E402
from tf_repos_b200.flags import FLAGS  # noqa: E402

flags.define_common(num_threads=10, embedding_size=256, batch_size=128, learning_rate=0.1, l2_reg=1.0,
                    deep_layers=None, dropout="1.0,0.5", batch_norm=False)      # AFM.py:41-53
flags.DEFINE_string("attention_layers", "256", "Attention Net mlp layers")      # AFM.py:52

def main():
    FLAGS._parse()
    from tf_repos_b200.afm import AFM
    from tf_repos_b200.estimator import run
    run(lambda: AFM(FLAGS.field_size, FLAGS.feature_size, FLAGS.embedding_size, FLAGS.batch_size,
                    attention_layers=FLAGS.attention_layers, dropout=FLAGS.dropout, l2_reg=FLAGS.l2_reg,
                    learning_rate=FLAGS.learning_rate, optimizer=FLAGS.optimizer, update_mode=FLAGS.update_mode), "AFM")


if __name__ == "__main__":
    main()
