"""Drop-in alias: `import COTR...` resolves to the H100-native implementation in `cotr_b200`.

The reference's demos (e.g. demo_single_pair.py) do
    from COTR.utils import utils, debug_utils
    from COTR.models import build_model
    from COTR.options.options import *
    from COTR.options.options_utils import *
    from COTR.inference.inference_helper import triangulate_corr
    from COTR.inference.sparse_engine import SparseEngine
With this repository root on sys.path those imports bind to cotr_b200 without touching the scripts.
"""
import importlib
import sys

_SUBMODULES = (
    "utils", "utils.utils", "utils.constants", "utils.debug_utils",
    "global_configs", "options", "options.options_utils", "options.options",
    "models", "models.misc", "models.cotr_model",
    "inference", "inference.inference_helper", "inference.refinement_task", "inference.sparse_engine",
)

for _name in _SUBMODULES:
    _mod = importlib.import_module("cotr_b200." + _name)
    sys.modules[__name__ + "." + _name] = _mod
    _parent, _, _leaf = _name.rpartition(".")
    if not _parent:
        setattr(sys.modules[__name__], _leaf, _mod)
