"""trieste_b200 — H100-native batched GP-posterior + acquisition engine behind trieste's
``ProbabilisticModel`` / ``AcquisitionFunctionBuilder`` / ``AcquisitionOptimizer`` interfaces.

Hand-written sm_90a CUDA behind a C-ABI (``include/trieste_b200.h``); no CPU fallback."""
from . import _lib  # noqa: F401
from .data import Dataset  # noqa: F401
from .kernels import RBF, Constant, Matern12, Matern32, Matern52, SquaredExponential  # noqa: F401
from .models import GaussianProcessRegression, GPRSpec, ModelStack, TrainableModelStack, build_gpr  # noqa: F401
from .space import Box, DiscreteSearchSpace, TaggedMultiSearchSpace  # noqa: F401

__version__ = "0.1.0"
