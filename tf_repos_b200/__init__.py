"""tf_repos_b200 -- H100-native (sm_90a) CTR feature-interaction engine; drop-in for the hot path of
lambdaji/tf_repos deep_ctr/Model_pipeline (see DESIGN.md).  Importing the package loads
libctr_b200.so and fails loudly if it has not been built."""
from . import _lib  # noqa: F401  (raises CtrError when the CUDA library is missing)

__all__ = ["_lib"]
