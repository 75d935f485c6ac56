#!/usr/bin/env python
"""Drop-in for DeepMTL/Model_pipeline/DeepCvrMTL.py (ESMM) on the H100 engine: same flags (DeepCvrMTL.py:34-60), TFRecord
input (`data_dir/tr/*tfrecord`, `data_dir/te/*tfrecord`), task types {train, eval, infer, export}, e.g.
  python Model_pipeline/DeepCvrMTL.py --task_type=train --field_size=11 --feature_size=4519540 --embedding_size=16 \
      --deep_layers=256,128 --dropout=0.8,0.5 --ctr_task_wgt=0.3 --l2_reg=0.005 --batch_size=1024 --num_epochs=1 \
      --model_dir=./model_ckpt/aliccp/ESMM/ --data_dir=./data/aliccp/"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tf_repos_b200 import flags  # noqa: E402
from tf_repos_b200.flags import FLAGS  # noqa: E402

flags.define_common(embedding_size=32, batch_size=64, checkpoint_format=False)
flags.DEFINE_float("ctr_task_wgt", 0.5, "loss weight of ctr task")     # DeepCvrMTL.py:49


def main():
    FLAGS._parse()
    from tf_repos_b200.esmm_main import run
    run()


if __name__ == "__main__":
    main()
