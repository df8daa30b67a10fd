"""diff-sampler_b200 — CUDA-native (H100, sm_90a) diffusion ODE sampling hot path (see DESIGN.md).

The directory name follows the repo layout contract; import it as `diff_sampler_b200`
(the sibling alias package extends its search path to this directory)."""
__version__ = '0.1'
