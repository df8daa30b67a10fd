"""The optimal (empirical-Bayes) denoiser of a dataset, natively: diff-analyzer's `get_denoised_opt` / `optimal_sampler`
(diff-analyzer-main/solvers.py:19-28, :773-868) and the nearest-neighbour read-out of its notebooks.

For a dataset y_0 .. y_{N-1} (rows of D = C*H*W values) the denoiser is

    D*(x; sigma) = sum_i softmax_i(-||x - y_i||^2 / (2 sigma^2)) y_i = sum_i softmax_i(u_i / sigma^2) y_i,   u_i = x.y_i - 0.5||y_i||^2

(-0.5||x||^2 is the same for every key and drops out of the softmax).  It is attention with one query per image, head dim D and N
keys, and runs as two tensor-core GEMMs with a row softmax between them (csrc/optimal.cu; numerics and bounds in DESIGN.md 4.9):

  1. opt_prep:     x -> fp16 hi/lo planes [2][B][D64] and ||x||^2 (fp64).
  2. GEMM (rows):  K-slice partials of x.y_i, one fp32 accumulator per 256-channel slice (z = slice), fp16x3.
  3. opt_softmax:  slices added in order in fp64, 0.5||y_i||^2 (fp64, packed once) subtracted; rows with a large logit error bound
                   rescored from exact distances; P = 2^15 softmax as fp16 hi/lo planes [2][B][N64].
  4. GEMM (rows):  split-K partials of P.Y over 2048-key chunks (z = chunk), fp16x3, against the transposed dataset planes.
  5. opt_reduce:   chunks added in order, times 2^-15, into D (NCHW fp32).

No atomics anywhere: two calls on the same input are bit-identical.
"""
import ctypes as C
import math

import torch

from . import _cstructs as S
from . import _lib
from . import gemm_desc as G
from .plan import F4, H2, NPL, PlanBuilder, WeightBlob, _align, io
from .solver_utils import get_schedule, solver_update

SLICE = 256                 # channels per fp32 accumulator of the logits GEMM (the error bound grows with the slice, DESIGN.md 4.9)
KEYS_PER_SPLIT = 2048       # dataset rows per split-K partial of the weighted sum
MAX_CHUNK = 512             # rows per plan run
WORKSPACE_BYTES = 2 << 30   # per-plan workspace bound: the batch is cut into chunks of at most this much workspace


def _pad(n, a=64):
    return -(-int(n) // a) * a


class _Geometry:
    """Shapes of the two contractions for a dataset of N rows of D values."""

    def __init__(self, N, D):
        self.N, self.D = N, D
        self.Dp, self.Np = _pad(D), _pad(N)             # fp16 plane pitches (64-element rows: 16-byte TMA strides, whole K blocks)
        self.Dq = _pad(D, 4)                            # pitch of the weighted-sum partials (vector stores of the GEMM epilogue)
        self.slice_c = min(SLICE, self.Dp)
        self.nslice = -(-self.Dp // self.slice_c)
        self.nsplit = -(-N // KEYS_PER_SPLIT)
        self.ksplit = _pad(-(-N // self.nsplit))
        self.nsplit = -(-N // self.ksplit)

    def row_bytes(self):
        """Workspace per batch row: logits partials, P planes, weighted-sum partials, x planes, ||x||^2."""
        return self.nslice * self.Np * F4 + NPL * self.Np * H2 + self.nsplit * self.Dq * F4 + NPL * self.Dp * H2 + 8

    def chunk(self):
        c = min(MAX_CHUNK, max(1, WORKSPACE_BYTES // self.row_bytes()))
        return c - c % 128 if c >= 128 else c          # whole 128-row M tiles


def compile_plan(g, wb, B, nsig, ymax, knn=0):
    """Lower one evaluation for B rows (nsig in {1, B} sigma values).  knn > 0: the nearest-neighbour read-out instead (dist / idx in
    the io slots D / BOTTLENECK).  Io slots: X = x [B][D], SIGMA, D = the denoiser output, BOTTLENECK = the per-row status (int32)."""
    assert nsig in (1, B)
    pb = PlanBuilder(wb, B, npass=3)
    W = wb.ref
    pb.need('xpl', NPL * B * g.Dp * H2)
    pb.need('xn2', B * 8)
    pb.need('part', g.nslice * B * g.Np * F4)
    pb.emit(lambda R: S.OptPrepDesc(x=io(S.DS_IO_X), planes=R('xpl'), xn2=R('xn2'), B=B, D=g.D, pitch=g.Dp))
    pb.emit(lambda R: G.rows_gemm(R('xpl'), B, g.Dp, 1, W('yrow'), g.N, g.Dp, 1, g.slice_c, num_z=g.nslice, nh=g.nslice, m_valid=B,
                                  n_valid=g.N, npass=3, a_c_per_zh=g.slice_c, b_k_per_zh=g.slice_c, out_f32=R('part'), o_zh=B * g.Np,
                                  ldo=g.Np, a_k_valid=g.D, b_k_valid=g.D)[0])
    common = lambda R: dict(part=R('part'), hy2=W('hy2'), xn2=R('xn2'), x=io(S.DS_IO_X), y=W('yf32'), ldp=g.Np, B=B, N=g.N, D=g.D,
                            nslice=g.nslice, ymax=ymax)
    if knn:
        pb.emit(lambda R: S.OptKnnDesc(dist=io(S.DS_IO_D), idx=io(S.DS_IO_BOTTLENECK), k=knn, **common(R)))
        return pb.finish(B=B, knn=knn)
    pb.need('P', NPL * B * g.Np * H2)
    pb.need('part2', g.nsplit * B * g.Dq * F4)
    pb.emit(lambda R: S.OptSoftmaxDesc(sigma=io(S.DS_IO_SIGMA), P=R('P'), status=io(S.DS_IO_BOTTLENECK), ldP=g.Np, nsig=nsig, **common(R)))
    pb.emit(lambda R: G.rows_gemm(R('P'), B, g.Np, 1, W('ycol'), g.D, g.Np, 1, g.ksplit, num_z=g.nsplit, nh=g.nsplit, m_valid=B,
                                  n_valid=g.D, npass=3, a_c_per_zh=g.ksplit, b_k_per_zh=g.ksplit, out_f32=R('part2'), o_zh=B * g.Dq,
                                  ldo=g.Dq, a_k_valid=g.N, b_k_valid=g.N)[0])
    pb.emit(lambda R: S.OptReduceDesc(part=R('part2'), out=io(S.DS_IO_D), rows=B, cols=g.D, ld=g.Dq, nsplit=g.nsplit,
                                      scale=2.0 ** -S.DS_OPT_P_SHIFT))
    return pb.finish(B=B, nsig=nsig)


def blob_layout(g):
    """Byte offsets of the packed dataset: row planes [2][N][Dp] fp16, transposed planes [2][D][Np] fp16, rows fp32 [N][D] (rescoring
    and exact distances), 0.5||y_i||^2 fp64 [N].  Returns (WeightBlob with the offsets, total bytes)."""
    wb = WeightBlob()
    size = 0
    for name, nbytes in (('yrow', NPL * g.N * g.Dp * H2), ('ycol', NPL * g.D * g.Np * H2), ('yf32', g.N * g.D * F4), ('hy2', g.N * 8)):
        size = _align(size)
        wb.off[name] = size
        size += nbytes
    wb.size = size
    return wb, size


def pack_dataset(y, g):
    """y: [N, D] fp32 (any device) -> (uint8 CPU blob, WeightBlob with the offsets, max ||y_i||)."""
    wb, size = blob_layout(g)
    blob = torch.zeros(size, dtype=torch.uint8)

    def put(name, t):
        t = t.contiguous().cpu()
        n = t.numel() * t.element_size()
        blob[wb.off[name]:wb.off[name] + n] = t.reshape(-1).view(torch.uint8)
    rows = torch.zeros(g.N, g.Dp, dtype=torch.float32, device=y.device)
    rows[:, :g.D] = y
    put('yrow', G.split_planes(rows))
    del rows
    cols = torch.zeros(g.D, g.Np, dtype=torch.float32, device=y.device)
    cols[:, :g.N] = y.t()
    put('ycol', G.split_planes(cols))
    del cols
    put('yf32', y)
    y2 = (y.double() ** 2).sum(dim=1)
    put('hy2', 0.5 * y2)
    return blob, wb, float(y2.max().sqrt()) * (1 + 1e-6)


class B200OptimalDenoiser:
    """D*(x; sigma) of a dataset [N, C, H, W] behind the `net(x, sigma)` contract of the native samplers (solvers.py), plus
    `nearest(x, k)`.  The dataset is packed once: fp16 hi/lo planes row-major and transposed, the fp32 rows and 0.5||y||^2
    (for CIFAR-10, 50 000 x 3 x 32 x 32: 1.23 GB of planes + 614 MB of fp32 rows).

    Batches larger than one chunk (at most 512 rows and at most WORKSPACE_BYTES = 2 GiB of workspace per plan) run as several plan
    launches.  Diagnostics of the last call: `last_row_status` ([B] int32: 0 GEMM logits, 1 rescored, 2 needed rescoring but the band
    exceeded the cap) and `last_unrefined_rows` (the count of 2s)."""

    label_dim = 0

    def __init__(self, dataset, device=None, sigma_min=0.002, sigma_max=80.0, cuda_graph=None):
        if not torch.is_tensor(dataset) or dataset.dim() != 4 or not dataset.is_floating_point():
            raise ValueError('dataset must be a floating-point [N, C, H, W] tensor')
        N, Cc, H, Wd = (int(v) for v in dataset.shape)
        if min(N, Cc, H, Wd) < 1:
            raise ValueError(f'empty dataset shape {tuple(dataset.shape)}')
        if N >= 2 ** 31 - 64 or Cc * H * Wd >= 2 ** 31 - 64:
            raise ValueError('dataset dimensions must fit in int32')
        self.device = torch.device(device) if device is not None else (dataset.device if dataset.is_cuda else torch.device('cuda'))
        if self.device.type != 'cuda':
            raise _lib.DsError('B200OptimalDenoiser needs a CUDA device (no CPU fallback)')
        if self.device.index is None:
            self.device = torch.device('cuda', torch.cuda.current_device())
        self.shape = (Cc, H, Wd)
        self.img_channels, self.img_resolution = Cc, H
        self.sigma_min, self.sigma_max = float(sigma_min), float(sigma_max)
        self.g = _Geometry(N, Cc * H * Wd)
        self.chunk = self.g.chunk()
        _, blob_bytes = blob_layout(self.g)
        need = blob_bytes + self.chunk * self.g.row_bytes()
        free, _total = torch.cuda.mem_get_info(self.device)
        if need > free:
            raise _lib.DsError(f'dataset does not fit: {need / 2**30:.2f} GiB needed (packed dataset + workspace), {free / 2**30:.2f} GiB free')
        y = dataset.detach().to(device=self.device, dtype=torch.float32).reshape(N, -1).contiguous()
        if not bool(torch.isfinite(y).all()):
            raise ValueError('dataset contains non-finite values')
        blob, self.wb, self.ymax = pack_dataset(y, self.g)
        del y
        self.native = _lib.NativePlans((C.c_ubyte * blob.numel()).from_address(blob.data_ptr()), self.device)
        del blob
        self.weight_bytes = blob_bytes
        from .net import default_cuda_graph
        self.cuda_graph = default_cuda_graph() if cuda_graph is None else bool(cuda_graph)
        self.last_row_status = None
        self.launches_last_forward = 0
        self.total_launches = 0

    @property
    def last_unrefined_rows(self):
        s = self.last_row_status
        return 0 if s is None else int((s == S.DS_OPT_UNREFINED).sum())

    def _plan(self, B, nsig, knn=0):
        g = self.g
        if knn:
            io_bytes = lambda pl: (B * g.D * 4, B * knn * 4, 0, 0, B * knn * 4, 0)
        else:
            io_bytes = lambda pl: (B * g.D * 4, B * g.D * 4, nsig * 4, 0, B * 4, 0)
        return self.native.get((B, nsig, knn), lambda: compile_plan(g, self.wb, B, nsig, self.ymax, knn),
                               io_bytes if self.cuda_graph else None)

    def _input(self, x):
        if not torch.is_tensor(x) or x.device.type != 'cuda':
            raise _lib.DsError('B200OptimalDenoiser: input must live on the CUDA device (no CPU fallback)')
        if x.dim() != 4 or tuple(x.shape[1:]) != self.shape:
            raise ValueError(f'x must be [B, {", ".join(map(str, self.shape))}], got {tuple(x.shape)}')
        if x.device != self.device:
            raise ValueError(f'x is on {x.device}, the dataset on {self.device}')
        return x.to(torch.float32).contiguous()

    def __call__(self, x, sigma, class_labels=None, out=None, **_):
        x = self._input(x)
        B = x.shape[0]
        sig = torch.as_tensor(sigma, dtype=torch.float32, device=x.device).reshape(-1).contiguous()
        if sig.numel() not in (1, B):
            raise ValueError(f'sigma must have 1 or {B} elements, got {sig.numel()}')
        per_sample = sig.numel() == B and B > 1
        if out is None:
            out = torch.empty_like(x)
        elif out.shape != x.shape or out.dtype != torch.float32 or not out.is_contiguous() or out.device != x.device:
            raise ValueError('out must be a contiguous float32 tensor shaped like x on the same device')
        status = torch.empty(B, dtype=torch.int32, device=x.device)
        stream = torch.cuda.current_stream(x.device).cuda_stream
        launches = 0
        for c0 in range(0, B, self.chunk):
            c1 = min(B, c0 + self.chunk)
            s = sig[c0:c1] if per_sample else sig
            nsig = s.numel() if s.numel() > 1 else 1
            h, _pl = self._plan(c1 - c0, nsig)
            launches += self.native.run(h, (x[c0].data_ptr(), out[c0].data_ptr(), s.data_ptr(), None, status[c0].data_ptr(), None), stream)
        self.last_row_status = status
        self.launches_last_forward = launches
        self.total_launches += launches
        return out

    def nearest(self, x, k):
        """(distances [B, k] fp32, indices [B, k] int64) of the k nearest dataset rows of each x (Euclidean, ascending, ties to the lower
        index), k <= 64: the KNN read-out of diff-analyzer's notebooks."""
        x = self._input(x)
        k = int(k)
        if not 1 <= k <= min(S.DS_KNN_MAX, self.g.N):
            raise ValueError(f'k must be in [1, {min(S.DS_KNN_MAX, self.g.N)}], got {k}')
        B = x.shape[0]
        dist = torch.empty(B, k, dtype=torch.float32, device=x.device)
        idx = torch.empty(B, k, dtype=torch.int32, device=x.device)
        stream = torch.cuda.current_stream(x.device).cuda_stream
        for c0 in range(0, B, self.chunk):
            c1 = min(B, c0 + self.chunk)
            h, _pl = self._plan(c1 - c0, 1, knn=k)
            self.native.run(h, (x[c0].data_ptr(), dist[c0].data_ptr(), None, None, idx[c0].data_ptr(), None), stream)
        return dist, idx.long()

    def profile_forward(self, x, sigma):
        """One evaluation of a single-chunk batch with per-op CUDA-event timing: list of (op type, ms)."""
        x = self._input(x)
        B = x.shape[0]
        if B > self.chunk:
            raise ValueError(f'profile_forward takes at most one chunk ({self.chunk} rows)')
        sig = torch.as_tensor(sigma, dtype=torch.float32, device=x.device).reshape(-1)
        self(x, sig)
        h, pl = self._plan(B, sig.numel() if sig.numel() > 1 else 1)
        lib = self.native.lib
        _lib.check(lib.ds_unet_set_profiling(h, 1), 'ds_unet_set_profiling')
        self(x, sig)
        buf = (C.c_float * pl.n_ops)()
        n = lib.ds_unet_get_profile(h, buf, pl.n_ops)
        lib.ds_unet_set_profiling(h, 0)
        return [(lib.ds_unet_op_type(h, i), float(buf[i])) for i in range(n)]

    def round_sigma(self, sigma):
        return torch.as_tensor(sigma)

    def eval(self):
        return self

    def to(self, *_a, **_k):
        return self

    def requires_grad_(self, *_a, **_k):
        return self


# ------------------------------------------------------------------------------------------------ drop-in functions
_CACHE = {}


def _dataset_key(ds):
    return (ds.device, ds.data_ptr(), tuple(ds.shape), tuple(ds.stride()), ds.dtype, ds._version)


def denoiser_for(dataset, device=None):
    """The B200OptimalDenoiser of `dataset`, packed once and reused while the tensor's storage, shape and version counter are
    unchanged (an in-place write bumps the version and re-packs).  At most one dataset is kept."""
    key = _dataset_key(dataset) + (str(device),)
    den = _CACHE.get(key)
    if den is None:
        _CACHE.clear()
        den = B200OptimalDenoiser(dataset, device=device)
        _CACHE[key] = den
    return den


@torch.no_grad()
def get_denoised_opt(x, t, cifar10_dataset):
    """Optimal denoiser output for the batch x at noise level t (reference: diff-analyzer-main/solvers.py:19-28)."""
    return denoiser_for(cifar10_dataset, device=x.device if x.is_cuda else None)(x, t)


@torch.no_grad()
def optimal_sampler(net, latents, cifar10_dataset, class_labels=None, num_steps=None, sigma_min=0.002, sigma_max=80,
                    schedule_type='polynomial', schedule_rho=7, afs=False, denoise_to_zero=False, return_inters=False,
                    return_denoised=False, return_eps=False, t_steps=None, **kwargs):
    """Euler sampler on the optimal denoiser of `cifar10_dataset` (reference: diff-analyzer-main/solvers.py:773-868).  `net` only
    feeds get_schedule (the 'discrete' schedule reads it).  Same return convention: x_N, or with return_inters the triple
    (trajectory [n (+1), B, ...], denoised [n - 1 (+1), ...], d [n - 1 (+1), ...]).

    Reference behaviour kept on purpose:
      * denoise_to_zero evaluates the denoiser at the LAST step's input x_{n-2} and sigma t_{n-2}, appends that denoised image to the
        trajectory and d = (x_{n-1} - denoised) / t_{n-1} to the eps list; without return_inters the result is still x_{n-1}.
    Reference failures turned into errors up front:
      * afs=True with return_denoised=True (the AFS step has no denoised image: UnboundLocalError in the reference);
      * return_inters=True without both return_denoised and return_eps (torch.cat of an empty list in the reference)."""
    if afs and return_denoised:
        raise ValueError('optimal_sampler: afs=True has no denoised image for the first step; return_denoised=True is not supported with it')
    if return_inters and not (return_denoised and return_eps):
        raise ValueError('optimal_sampler: return_inters=True returns (trajectory, denoised, eps) and needs return_denoised=True and '
                         'return_eps=True')
    if latents.device.type != 'cuda':
        raise RuntimeError('optimal_sampler: latents must be on a CUDA device (there is no CPU fallback)')
    den = denoiser_for(cifar10_dataset, device=latents.device)
    if t_steps is None:
        t_steps = get_schedule(num_steps, sigma_min, sigma_max, device=latents.device, schedule_type=schedule_type,
                               schedule_rho=schedule_rho, net=net)
    t = [float(v) for v in t_steps.reshape(-1).tolist()]
    n = len(t)
    lat = latents.to(torch.float32).contiguous()
    shape = tuple(lat.shape)
    extra = 1 if denoise_to_zero else 0
    xt = torch.empty((n + extra,) + shape, device=lat.device) if return_inters else None
    dens = torch.empty((n - 1 + extra,) + shape, device=lat.device) if return_inters else None
    eps = torch.empty((n - 1 + extra,) + shape, device=lat.device) if return_inters else None
    bufs = None if return_inters else (torch.empty_like(lat), torch.empty_like(lat))
    x = xt[0] if return_inters else bufs[0]
    solver_update(x, lat, [t[0]], mode=S.DS_M_NONE)                          # x_next = latents * t_steps[0]
    dbuf = None if return_inters else torch.empty_like(lat)
    D, x_cur = None, x
    for i in range(n - 1):
        x_cur = x
        out = xt[i + 1] if return_inters else bufs[(i + 1) % 2]
        h = t[i + 1] - t[i]
        if afs and i == 0:                                                   # AFS: d = x / sqrt(1 + t^2), no evaluation
            solver_update(out, x_cur, [1.0, h], mode=S.DS_M_DIV, t=math.sqrt(1.0 + t[i] * t[i]))
            D = None
        else:
            D = den(x_cur, t[i], out=dens[i] if return_inters else dbuf)
            solver_update(out, x_cur, [1.0, h], mode=S.DS_M_EPS, D=D, t=t[i], out_m=eps[i] if return_inters else None)
        x = out
    if denoise_to_zero and return_inters:                                    # without return_inters the reference returns x_{n-1}
        xt[n].copy_(D)
        dens[n - 1].copy_(D)
        solver_update(eps[n - 1], x, [0.0, 1.0], mode=S.DS_M_EPS, D=D, t=t[n - 1])
    if return_inters:
        return xt, dens, eps
    return x
