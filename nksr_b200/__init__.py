"""nksr_b200 -- H100-native implementation of the NKSR reconstruction hot path.

Same Python surface as the reference's closed `nksr` wheel (SURVEY.md Appendix A):
Reconstructor, SparseFeatureHierarchy, NKSRNetwork, fields.{KernelField, NeuralField,
LayerField, PCNNField}, configs.load_checkpoint_from_url, get_estimate_normal_preprocess_fn.
All arithmetic of the hot path runs in hand-written sm_90a CUDA kernels behind the C-ABI of
include/nksr_b200.h (nksr_b200/libnksr_b200.so); there is no CPU or PyTorch fallback.
Inference only: the solve is not differentiable (the reference needs that for training only).
"""
from . import _lib, fields, meshing, network, sdfgen, svh  # noqa: F401
from .fields import KernelField, LayerField, NeuralField, PCNNField  # noqa: F401
from .network import NKSRNetwork, load_checkpoint_from_url  # noqa: F401
from .reconstructor import Reconstructor, get_estimate_normal_preprocess_fn  # noqa: F401
from .svh import SparseFeatureHierarchy  # noqa: F401

__version__ = "0.1.0"


class _Configs:
    load_checkpoint_from_url = staticmethod(load_checkpoint_from_url)


configs = _Configs()
utils = network  # `from nksr import utils` is imported (unused) at examples/recons_colored_mesh.py:12
