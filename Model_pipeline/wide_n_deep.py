#!/usr/bin/env python
"""Drop-in for deep_ctr/Model_pipeline/wide_n_deep.py on the H100 engine: same flags (wide_n_deep.py:21-47), same
CSV input (tr*csv / va*csv / te*csv, 40 columns), same task types {train, predict, export_model}, e.g.
  python Model_pipeline/wide_n_deep.py --model_type=wide_n_deep --num_epochs=1 --batch_size=128 \
      --model_dir=./model_ckpt/criteo/wide_n_deep/ --data_dir=./data/criteo/"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tf_repos_b200 import flags  # noqa: E402
from tf_repos_b200.flags import FLAGS  # noqa: E402

flags.DEFINE_boolean("dist_mode", False, "run use distribuion mode or not")
flags.DEFINE_string("ps_hosts", "", "Comma-separated list of hostname:port pairs")
flags.DEFINE_string("worker_hosts", "", "Comma-separated list of hostname:port pairs")
flags.DEFINE_string("job_name", "", "One of 'ps', 'worker'")
flags.DEFINE_integer("task_index", 0, "Index of task within the job")
flags.DEFINE_integer("num_threads", 10, "Number of threads")
flags.DEFINE_integer("embedding_size", 32, "Embedding size")
flags.DEFINE_integer("num_epochs", 10, "Number of epochs")
flags.DEFINE_integer("batch_size", 128, "batch size")
flags.DEFINE_string("deep_layers", "256,128,64", "deep layers")
flags.DEFINE_integer("log_steps", 1000, "save summary every steps")
flags.DEFINE_integer("throttle_secs", 600, "evaluate every 10mins")
flags.DEFINE_string("data_dir", "", "data dir")
flags.DEFINE_string("dt_dir", "", "data dt partition")
flags.DEFINE_string("model_dir", "", "model check point dir")
flags.DEFINE_string("servable_model_dir", "", "export servable model for TensorFlow Serving")
flags.DEFINE_string("task_type", "train", "task type {train, predict, export}")
flags.DEFINE_string("model_type", "wide_n_deep", "model type {'wide', 'deep', 'wide_n_deep'}")
flags.DEFINE_boolean("clear_existing_model", False, "clear existing model or not")


def main():
    FLAGS._parse()
    from tf_repos_b200.wide_deep_main import run
    run()


if __name__ == "__main__":
    main()
