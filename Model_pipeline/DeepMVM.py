#!/usr/bin/env python
"""Drop-in for deep_ctr/Model_pipeline/DeepMVM.py on the H100 engine (flags: DeepMVM.py:35-60, no model-specific flag;
--loss_type is accepted and, as in the reference, unused)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tf_repos_b200 import flags  # noqa: E402
from tf_repos_b200.flags import FLAGS  # noqa: E402

flags.define_common()


def main():
    FLAGS._parse()
    from tf_repos_b200.deepmvm import DeepMVM
    from tf_repos_b200.estimator import run
    run(lambda: DeepMVM(FLAGS.field_size, FLAGS.feature_size, FLAGS.embedding_size, FLAGS.batch_size,
                        deep_layers=FLAGS.deep_layers, dropout=FLAGS.dropout, l2_reg=FLAGS.l2_reg,
                        learning_rate=FLAGS.learning_rate, optimizer=FLAGS.optimizer, update_mode=FLAGS.update_mode,
                        batch_norm=FLAGS.batch_norm, batch_norm_decay=FLAGS.batch_norm_decay), "DeepMVM")


if __name__ == "__main__":
    main()
