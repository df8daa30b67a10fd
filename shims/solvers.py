"""Import shim: lets the reference's `import solvers` resolve to the CUDA-native implementation (see INTEGRATION.md)."""
from diff_sampler_b200.solvers import *          # noqa: F401,F403
from diff_sampler_b200 import solvers as _impl

globals().update({k: v for k, v in vars(_impl).items() if not k.startswith('__')})
