"""Import shim: lets the reference's `import solver_utils` resolve to the CUDA-native implementation (see INTEGRATION.md)."""
from diff_sampler_b200.solver_utils import *          # noqa: F401,F403
from diff_sampler_b200 import solver_utils as _impl

globals().update({k: v for k, v in vars(_impl).items() if not k.startswith('__')})
