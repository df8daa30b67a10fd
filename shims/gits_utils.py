"""Import shim: lets the reference's `import gits_utils` resolve to the CUDA-native implementation (see INTEGRATION.md)."""
from diff_sampler_b200.gits_utils import *          # noqa: F401,F403
from diff_sampler_b200 import gits_utils as _impl

globals().update({k: v for k, v in vars(_impl).items() if not k.startswith('__')})
