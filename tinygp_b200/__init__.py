"""tinygp_b200 -- an H100-native (sm_90a) solver backend behind tinygp's plugin surface.

``GaussianProcess`` / ``kernels`` / ``noise`` / ``solvers`` mirror ``tinygp``'s names
(src/tinygp/__init__.py); the arithmetic runs in hand-written sm_90a CUDA behind the C-ABI of
``include/b200gp.h``.  There is no CPU fallback.  ``adapter.DirectSolver`` / ``adapter.QuasisepSolver`` accept the
reference's own kernel / noise objects and can be passed as ``solver=`` to ``tinygp.GaussianProcess``.
"""

__version__ = "0.1.0"

from tinygp_b200 import (
    adapter as adapter,
    kernels as kernels,
    means as means,
    noise as noise,
    solvers as solvers,
    transforms as transforms,
)
from tinygp_b200.gp import ConditionResult as ConditionResult, GaussianProcess as GaussianProcess
