"""ctypes binding of include/diffsampler_b200.h.  There is no CPU fallback: if the shared library is
missing or a call fails, this raises."""
import ctypes as C
import os

import torch

from . import _cstructs as S

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libdiffsampler_b200.so')

EXPORTS = [
    'ds_version', 'ds_last_error', 'ds_weights_create', 'ds_weights_destroy', 'ds_unet_create', 'ds_unet_destroy',
    'ds_unet_forward', 'ds_unet_debug_read', 'ds_unet_last_launch_count', 'ds_solver_update', 'ds_dyn_threshold',
    'ds_op_launch', 'ds_sizeof', 'ds_unet_set_profiling', 'ds_unet_get_profile', 'ds_unet_op_type', 'ds_gits_cost', 'ds_unet_forward_io', 'ds_images_to_uint8', 'ds_solver_update_u8', 'ds_unet_enable_graph', 'ds_amed_predict',
    'ds_gemm_config', 'ds_op_check',
]

_lib = None


class DsError(RuntimeError):
    pass


def load():
    """Load (once) and type the library.  Raises if it has not been built (python -m diff_sampler_b200.build)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise DsError(f'{LIB_PATH} not found: build it with `python diff-sampler_b200/build.py` '
                      '(there is no CPU fallback for the CUDA path)')
    lib = C.CDLL(LIB_PATH)
    vp, cp, sz = C.c_void_p, C.c_char_p, C.c_size_t
    lib.ds_version.restype = cp
    lib.ds_last_error.restype = cp
    lib.ds_weights_create.argtypes = [vp, sz, C.POINTER(vp)]
    lib.ds_weights_destroy.argtypes = [vp]
    lib.ds_weights_destroy.restype = None
    lib.ds_unet_create.argtypes = [vp, vp, C.c_int, sz, sz, C.POINTER(vp)]
    lib.ds_unet_destroy.argtypes = [vp]
    lib.ds_unet_destroy.restype = None
    lib.ds_unet_forward.argtypes = [vp, vp, vp, vp, vp, vp, vp]
    lib.ds_unet_forward_io.argtypes = [vp, C.POINTER(vp), C.c_int, vp]
    lib.ds_unet_enable_graph.argtypes = [vp, C.POINTER(sz), C.c_int]
    lib.ds_unet_debug_read.argtypes = [vp, sz, vp, sz, vp]
    lib.ds_unet_last_launch_count.argtypes = [vp]
    lib.ds_unet_set_profiling.argtypes = [vp, C.c_int]
    lib.ds_unet_get_profile.argtypes = [vp, C.POINTER(C.c_float), C.c_int]
    lib.ds_unet_op_type.argtypes = [vp, C.c_int]
    lib.ds_solver_update.argtypes = [vp, vp, vp, vp, vp, C.POINTER(vp), C.c_int, vp, C.c_int, C.c_float, vp,
                                     C.POINTER(C.c_float), vp, C.c_int64, C.c_int, vp]
    lib.ds_solver_update_u8.argtypes = [vp, vp, vp, C.c_int, C.c_int, vp, vp, vp, C.POINTER(vp), C.c_int, vp, C.c_int, C.c_float, vp,
                                        C.POINTER(C.c_float), vp, C.c_int64, C.c_int, vp]
    lib.ds_amed_predict.argtypes = [vp, C.POINTER(C.c_int), vp, vp, vp, C.c_float, C.c_float, vp, C.c_int, vp]
    lib.ds_dyn_threshold.argtypes = [vp, vp, C.c_int, C.c_int, C.c_float, C.c_float, vp]
    lib.ds_gits_cost.argtypes = [vp, vp, vp, vp, C.c_int, C.c_int, C.c_int64, vp]
    lib.ds_images_to_uint8.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, vp]
    lib.ds_op_launch.argtypes = [C.c_int, vp, sz, vp]
    lib.ds_op_check.argtypes = [C.c_int, vp, sz]
    lib.ds_sizeof.argtypes = [C.c_int]
    lib.ds_sizeof.restype = sz
    lib.ds_gemm_config.argtypes = [vp, C.POINTER(C.c_int)]
    for which, cls in S.SIZEOF_CHECKS.items():
        got, want = C.sizeof(cls), lib.ds_sizeof(which)
        if got != want:
            raise DsError(f'struct mirror {cls.__name__}: ctypes size {got} != library size {want}')
    _lib = lib
    return lib


def check(rc, what=''):
    if rc != 0:
        msg = load().ds_last_error().decode()
        raise DsError(f'{what} failed (rc={rc}): {msg}')


def version():
    return load().ds_version().decode()


def op_launch(desc, stream=0):
    """Launch one kernel-level op from a descriptor struct holding absolute device pointers."""
    lib = load()
    check(lib.ds_op_launch(S.OP_TYPE_OF[type(desc)], C.byref(desc), C.sizeof(desc), C.c_void_p(stream)), type(desc).__name__)


def op_check(desc):
    """None if the launcher of the descriptor's op accepts it, else the rule it breaks ("<op>: <rule>").  Needs no GPU; pointer fields
    are only tested against NULL, so plan descriptors holding references are checked as they are."""
    lib = load()
    if lib.ds_op_check(S.OP_TYPE_OF[type(desc)], C.byref(desc), C.sizeof(desc)) == 0:
        return None
    return lib.ds_last_error().decode()


def gemm_config(desc):
    """How the GEMM kernel runs a GemmDesc on the current device: dict(stages, grid)."""
    info = (C.c_int * 2)()
    check(load().ds_gemm_config(C.byref(desc), info), 'ds_gemm_config')
    return dict(stages=info[0], grid=info[1])


class NativePlans:
    """One weight blob on a CUDA device (ds_weights_create) and the native plans compiled against it (ds_unet_create), keyed by the
    shape they were compiled for.  Destroys every handle when collected."""

    def __init__(self, blob, device):
        self.lib = load()
        self.device = device
        self.plans = {}                 # key -> (ds_unet handle, plan.Plan)
        self._wh = C.c_void_p()
        with torch.cuda.device(device):
            check(self.lib.ds_weights_create(blob, len(blob), C.byref(self._wh)), 'ds_weights_create')

    def get(self, key, compile_fn, io_bytes=None):
        """(handle, plan) for `key`; the plan is compile_fn() on first use.  io_bytes(plan) -> the byte sizes of the six io slots turns
        on CUDA-graph replay of every forward (ds_unet_enable_graph)."""
        ent = self.plans.get(key)
        if ent is None:
            pl = compile_fn()
            h = C.c_void_p()
            with torch.cuda.device(self.device):
                check(self.lib.ds_unet_create(self._wh, C.cast(pl.ops_array, C.c_void_p), pl.n_ops, C.sizeof(S.PlanOp), pl.arena_bytes,
                                              C.byref(h)), 'ds_unet_create')
                if io_bytes is not None:
                    check(self.lib.ds_unet_enable_graph(h, (C.c_size_t * S.DS_IO_COUNT)(*io_bytes(pl)), S.DS_IO_COUNT),
                          'ds_unet_enable_graph')
            ent = self.plans[key] = (h, pl)
        return ent

    def run(self, h, io, stream):
        """One forward of plan handle h over the io slots (device pointers or None, DS_IO_* order) on `stream`.
        Returns the number of kernels it launched."""
        check(self.lib.ds_unet_forward_io(h, (C.c_void_p * S.DS_IO_COUNT)(*io), S.DS_IO_COUNT, C.c_void_p(stream)), 'ds_unet_forward_io')
        return self.lib.ds_unet_last_launch_count(h)

    def debug_read(self, key, name, numel, dtype=torch.float32):
        """Copy the arena buffer `name` of the plan for `key` to the host (tests only)."""
        h, pl = self.plans[key]
        t = torch.empty(numel, dtype=dtype)
        stream = torch.cuda.current_stream(self.device).cuda_stream
        check(self.lib.ds_unet_debug_read(h, pl.arena_offsets[name], t.data_ptr(), t.numel() * t.element_size(), C.c_void_p(stream)),
              'ds_unet_debug_read')
        return t

    def __del__(self):
        try:
            for h, _ in self.plans.values():
                self.lib.ds_unet_destroy(h)
            self.lib.ds_weights_destroy(self._wh)
        except Exception:
            pass
