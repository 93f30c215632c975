"""Drop-in alias: `import nksr` resolves to the H100-native implementation (nksr_b200), so the
reference's examples/*.py and models/nksr_net.py import unchanged (SURVEY.md Appendix A)."""
import sys as _sys

import nksr_b200 as _impl
from nksr_b200 import *  # noqa: F401,F403
from nksr_b200 import (KernelField, LayerField, NeuralField, NKSRNetwork, PCNNField, Reconstructor,  # noqa: F401
                       SparseFeatureHierarchy, configs, fields, get_estimate_normal_preprocess_fn, svh, utils)

_sys.modules[__name__ + ".fields"] = _impl.fields
_sys.modules[__name__ + ".svh"] = _impl.svh
_sys.modules[__name__ + ".configs"] = _impl.configs
_sys.modules[__name__ + ".utils"] = _impl.network
