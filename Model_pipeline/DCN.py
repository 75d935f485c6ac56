#!/usr/bin/env python
"""Drop-in for deep_ctr/Model_pipeline/DCN.py on the H100 engine (flags: DCN.py:29-58, incl. --cross_layers)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tf_repos_b200 import flags  # noqa: E402
from tf_repos_b200.flags import FLAGS  # noqa: E402

flags.define_common(loss_type=False)
flags.DEFINE_integer("cross_layers", 3, "cross layers, polynomial degree")


def main():
    FLAGS._parse()
    from tf_repos_b200.dcn import DCN
    from tf_repos_b200.estimator import run
    run(lambda: DCN(FLAGS.field_size, FLAGS.feature_size, FLAGS.embedding_size, FLAGS.batch_size,
                    deep_layers=FLAGS.deep_layers, cross_layers=FLAGS.cross_layers, dropout=FLAGS.dropout,
                    l2_reg=FLAGS.l2_reg, learning_rate=FLAGS.learning_rate, optimizer=FLAGS.optimizer,
                    update_mode=FLAGS.update_mode,
                 batch_norm=FLAGS.batch_norm, batch_norm_decay=FLAGS.batch_norm_decay), "DCN")


if __name__ == "__main__":
    main()
