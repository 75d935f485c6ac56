#!/usr/bin/env python
"""Drop-in for deep_ctr/Model_pipeline/DeepFM.py on the H100 engine: same flags (DeepFM.py:34-60), same
libsvm input, same task types.  e.g.
  python Model_pipeline/DeepFM.py --task_type=train --learning_rate=0.0005 --optimizer=Adam --num_epochs=1 \
      --batch_size=256 --field_size=39 --feature_size=117581 --deep_layers=400,400,400 --dropout=0.5,0.5,0.5 \
      --log_steps=1000 --num_threads=8 --model_dir=./model_ckpt/criteo/DeepFM/ --data_dir=./data/criteo/
(deep_ctr/run.sh:13)"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tf_repos_b200 import flags  # noqa: E402
from tf_repos_b200.flags import FLAGS  # noqa: E402

flags.define_common()


def main():
    FLAGS._parse()
    from tf_repos_b200.deepfm import DeepFM
    from tf_repos_b200.estimator import run
    run(lambda: DeepFM(FLAGS.field_size, FLAGS.feature_size, FLAGS.embedding_size, FLAGS.batch_size,
                       deep_layers=FLAGS.deep_layers, dropout=FLAGS.dropout, l2_reg=FLAGS.l2_reg,
                       learning_rate=FLAGS.learning_rate, optimizer=FLAGS.optimizer, update_mode=FLAGS.update_mode,
                 batch_norm=FLAGS.batch_norm, batch_norm_decay=FLAGS.batch_norm_decay),
        "DeepFM")


if __name__ == "__main__":
    main()
