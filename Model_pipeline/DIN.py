#!/usr/bin/env python
"""Drop-in for deep_ctr/Model_pipeline/DIN.py on the H100 engine: same flags (DIN.py:26-54), TFRecord input
(`data_dir/tr/*tfrecord`, `data_dir/te/*tfrecord`), task types {train, eval, infer, export}, e.g.
  python Model_pipeline/DIN.py --task_type=train --field_size=11 --feature_size=1000000 --embedding_size=32 \
      --batch_size=1024 --num_epochs=1 --model_dir=./model_ckpt/aliccp/DIN/ --data_dir=./data/aliccp/"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tf_repos_b200 import flags  # noqa: E402
from tf_repos_b200.flags import FLAGS  # noqa: E402

flags.define_common(embedding_size=32, batch_size=64)
flags.DEFINE_boolean("attention_pooling", True, "attention pooling")        # DIN.py:45
flags.DEFINE_string("attention_layers", "256", "Attention Net mlp layers")   # DIN.py:46


def main():
    FLAGS._parse()
    from tf_repos_b200.din_main import run
    run()


if __name__ == "__main__":
    main()
