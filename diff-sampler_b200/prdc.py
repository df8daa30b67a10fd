"""Precision, recall, density and coverage (and per-sample realism) of sfd-main/prdc.py (:29-125), natively.

With R the real rows, F the fake rows, k = nearest_k, r_i the (k+1)-th smallest distance of real row i to R (its own distance 0
included), s_j that of fake row j to F and d_ij = ||R_i - F_j||:

    precision = mean_j [exists i: d_ij < r_i]         recall   = mean_i [exists j: d_ij < s_j]
    density   = (1 / k) * mean_j #{i: d_ij < r_i}     coverage = mean_i [exists j: d_ij < r_i]
    realism_j = max over {i: r_i < median(r)} of r_i / d_ij

Every distance is float64, the square root of a float64 sum of squared float64 differences, and every comparison is on distances, as
the reference makes them; the scores are formed from integer counts in the reference's own operation order.  So the results are the
exact-arithmetic ones, bit for bit, wherever the reference's own distance matrices are exact (DESIGN.md 4.12).

Per query chunk (csrc/prdc.cu):
  1. GEMM (rows):  K-slice partials of the scaled q.t, one fp32 accumulator per 256-channel slice, fp16x3, against the other set's
                   row planes.
  2. prdc_kth:     the (k+1)-th smallest distance of each row to its own set (R x R once per real set, F x F per call), or
     prdc_count:   the neighbourhood counts: F x R gives precision, density and realism, R x F recall and coverage.
Pairs whose approximate distance lies within the GEMM's error bound of a threshold are recomputed exactly on the GPU; there is no cap.
No atomics anywhere: two calls on the same input are bit-identical.
"""
import ctypes as C
import math

import numpy as np
import torch

from . import _cstructs as S
from . import _lib
from . import gemm_desc as G
from .plan import F4, H2, NPL, PlanBuilder, WeightBlob

SLICE = 256                 # channels per fp32 accumulator of the distance GEMMs (the error bound grows with the slice, DESIGN.md 4.12)
WORKSPACE_BYTES = 2 << 30   # bound on the GEMM partials of one query chunk: the query rows are cut into chunks of at most this much
MAX_K = S.DS_PRDC_KMAX      # largest nearest_k: prdc_kth keeps the k + 1 best candidates of a row in shared memory


def _pad(n, a=64):
    return -(-int(n) // a) * a


class SetRefs:
    """Where one feature set of N rows of D values lives: fp16 hi/lo planes [2][N][Dp] of `scale` * rows (scale a power of two),
    the float64 rows [N][D], their squared norms [N], and the k-NN radii [N] with their exact squared distances [N].  Pointers are
    device addresses or plan references."""

    def __init__(self, N, D, planes, rows, n2, rad, rad2, scale=1.0):
        self.N, self.D, self.Dp = int(N), int(D), _pad(D)
        self.planes, self.rows, self.n2, self.rad, self.rad2 = planes, rows, n2, rad, rad2
        self.scale = float(scale)


def slices(D):
    """(channels per slice, slice count) of the distance GEMMs over D channels."""
    Dp = _pad(D)
    c = min(SLICE, Dp)
    return c, -(-Dp // c)


def chunk_rows(n_query, n_target, D):
    """Query rows per GEMM launch: the slice partials of a chunk stay within WORKSPACE_BYTES (whole 128-row M tiles)."""
    _, ns = slices(D)
    c = max(1, WORKSPACE_BYTES // (ns * _pad(n_target) * F4))
    c = c - c % 128 if c >= 128 else c
    return min(c, n_query)


def compile_plan(passes, D, k):
    """One plan running `passes` in order.  Each pass is
        ('kth', Q, nres)                               Q.rad / Q.rad2 <- the (k+1)-th distance of each row of Q to Q;
        ('count', Q, T, cnt_t, cnt_own, realism, med, nres)
                                                       counts of Q's rows against T with T's radii; cnt_own (or 0) against Q's own
                                                       radii; realism (or 0) over the targets with radius < med.
    Q / T are SetRefs; the other pointers are [Q.N] arrays (int32 counts, float64 realism; nres int32 or 0)."""
    slice_c, nslice = slices(D)
    pb = PlanBuilder(WeightBlob(), 1)
    for ps in passes:
        kind, Q = ps[0], ps[1]
        T = Q if kind == 'kth' else ps[2]
        Np = _pad(T.N)
        chunk = chunk_rows(Q.N, T.N, D)
        pb.need('part', nslice * chunk * Np * F4)
        for c0 in range(0, Q.N, chunk):
            B = min(chunk, Q.N - c0)

            def gemm(R, Q=Q, T=T, c0=c0, B=B, Np=Np):
                d, _ = G.rows_gemm(Q.planes + c0 * Q.Dp * H2, Q.N, Q.Dp, 1, T.planes, T.N, T.Dp, 1, slice_c, num_z=nslice, nh=nslice,
                                   m_valid=B, n_valid=T.N, npass=3, a_c_per_zh=slice_c, b_k_per_zh=slice_c, out_f32=R('part'),
                                   o_zh=B * Np, ldo=Np, a_k_valid=D, b_k_valid=D)
                d.a_dims[1] = B                 # the chunk's rows; the planes keep the whole set's plane stride
                return d
            pb.emit(gemm)
            common = lambda R, Q=Q, T=T, c0=c0, B=B, Np=Np: dict(
                part=R('part'), q=Q.rows + c0 * D * 8, t=T.rows, qn2=Q.n2 + c0 * 8, tn2=T.n2, ldp=Np, B=B, N=T.N, D=D, nslice=nslice,
                sq=Q.scale, st=T.scale)
            if kind == 'kth':
                nres = ps[2]
                pb.emit(lambda R, c=common, Q=Q, c0=c0, nres=nres: S.PrdcKthDesc(
                    rad=Q.rad + c0 * 8, rad2=Q.rad2 + c0 * 8, nres=nres + c0 * 4 if nres else 0, k=k, **c(R)))
            else:
                _, _, _, cnt_t, cnt_own, realism, med, nres = ps
                pb.emit(lambda R, c=common, Q=Q, T=T, c0=c0, cnt_t=cnt_t, cnt_own=cnt_own, realism=realism, med=med, nres=nres:
                        S.PrdcCountDesc(tau=T.rad, tau2=T.rad2, rho=Q.rad + c0 * 8 if cnt_own else 0, rho2=Q.rad2 + c0 * 8 if cnt_own else 0,
                                        cnt_t=cnt_t + c0 * 4, cnt_own=cnt_own + c0 * 4 if cnt_own else 0,
                                        realism=realism + c0 * 8 if realism else 0, med=med, nres=nres + c0 * 4 if nres else 0, **c(R)))
    return pb.finish(D=D, k=k)


def operand_scale(x):
    """The power of two that brings max |x| into [2^13, 2^14): the fp16 hi plane cannot overflow, and small features keep their
    precision above fp16's subnormal floor."""
    m = float(x.abs().max()) if x.numel() else 0.0
    if m == 0.0:
        return 1.0
    return math.ldexp(1.0, max(-300, min(300, 14 - math.frexp(m)[1])))


def split_rows(x, scale, Dp):
    """float64 rows [N, D] -> fp16 hi/lo planes [2][N][Dp] of fp32(scale * x), columns D.. zero."""
    v = torch.zeros(x.shape[0], Dp, dtype=torch.float32, device=x.device)
    v[:, :x.shape[1]] = (x * scale).float()
    return G.split_planes(v)


def _rows(x, name):
    """numpy array or torch tensor, fp32 or fp64, [N, D] -> float64 contiguous rows on its own device (fp32 widened, fp64 kept)."""
    if isinstance(x, np.ndarray):
        x = torch.from_numpy(x)
    if not torch.is_tensor(x):
        raise ValueError(f'{name} must be a numpy array or a torch tensor')
    if x.dtype not in (torch.float32, torch.float64):
        raise ValueError(f'{name} must be float32 or float64, got {x.dtype}')
    if x.dim() != 2 or min(x.shape) < 1:
        raise ValueError(f'{name} must be [N, D] with N, D >= 1, got {tuple(x.shape)}')
    if x.shape[0] >= 2 ** 31 - 64 or x.shape[1] >= 2 ** 31 - 64:
        raise ValueError(f'{name}: dimensions must fit in int32')
    x = x.detach().to(torch.float64).contiguous()
    if not bool(torch.isfinite(x).all()):
        raise ValueError(f'{name} contains non-finite values')
    return x


def _check_k(nearest_k):
    if isinstance(nearest_k, bool) or not isinstance(nearest_k, (int, np.integer)) or nearest_k < 1:
        raise ValueError(f'nearest_k must be an integer >= 1, got {nearest_k!r}')
    if nearest_k > MAX_K:
        raise ValueError(f'nearest_k must be at most {MAX_K} (the candidate cap of prdc_kth), got {nearest_k}')
    return int(nearest_k)


def _check_rows(x, k, name):
    if x.shape[0] < k + 2:
        raise ValueError(f'{name} has {x.shape[0]} rows; nearest_k = {k} needs at least {k + 2} (the (k+1)-th neighbour of each '
                         'row other than itself)')


class _DeviceSet:
    """A feature set's device buffers (SetRefs at their addresses); fill() replaces the rows in place, so plans stay valid."""

    def __init__(self, N, D, device):
        Dp = _pad(D)
        self.planes = torch.empty(NPL, N, Dp, dtype=torch.float16, device=device)
        self.rows = torch.empty(N, D, dtype=torch.float64, device=device)
        self.n2 = torch.empty(N, dtype=torch.float64, device=device)
        self.rad = torch.empty(N, dtype=torch.float64, device=device)
        self.rad2 = torch.empty(N, dtype=torch.float64, device=device)
        self.nres = torch.zeros(N, dtype=torch.int32, device=device)
        self.refs = SetRefs(N, D, self.planes.data_ptr(), self.rows.data_ptr(), self.n2.data_ptr(), self.rad.data_ptr(),
                            self.rad2.data_ptr())

    def fill(self, x):
        scale = operand_scale(x)
        self.rows.copy_(x)
        self.planes.copy_(split_rows(x, scale, self.refs.Dp))
        torch.sum(x * x, dim=1, out=self.n2)
        self.refs.scale = scale


class B200PRDC:
    """sfd-main/prdc.py's metrics against one real feature set, packed once and with its radii computed once; score() takes fake
    sets.  Inputs are numpy arrays or torch tensors, fp32 (widened to float64, as prdc.py's callers pass them) or fp64, [N, D].

    Query rows run in chunks whose GEMM partials stay within WORKSPACE_BYTES (2 GiB), so 50 000 x 50 000 x 2048 fits on one H100.
    cuda_graph (default: DSB_CUDA_GRAPH != '0') replays each plan as one CUDA graph.  Diagnostic: `last_rescored_pairs`, the number of
    pairs the last call recomputed exactly."""

    def __init__(self, real_features, nearest_k=5, device=None, cuda_graph=None):
        self.k = _check_k(nearest_k)
        x = _rows(real_features, 'real_features')
        _check_rows(x, self.k, 'real_features')
        if device is None:
            device = real_features.device if torch.is_tensor(real_features) and real_features.is_cuda else torch.device('cuda')
        self.device = torch.device(device)
        if self.device.type != 'cuda':
            raise _lib.DsError('B200PRDC needs a CUDA device (no CPU fallback)')
        if self.device.index is None:
            self.device = torch.device('cuda', torch.cuda.current_device())
        x = x.to(self.device)
        self.N, self.D = x.shape
        from .net import default_cuda_graph
        self.cuda_graph = default_cuda_graph() if cuda_graph is None else bool(cuda_graph)
        self.real = _DeviceSet(self.N, self.D, self.device)
        self.real.fill(x)
        del x
        self._native = _lib.NativePlans((C.c_ubyte * 1024)(), self.device)
        h, _ = self._plan(self._native, 'radii', lambda: compile_plan([('kth', self.real.refs, self.real.nres.data_ptr())], self.D, self.k))
        self._run(self._native, h)
        self.radii = self.real.rad.cpu().numpy()
        self.median = np.median(self.radii)
        self.last_rescored_pairs = int(self.real.nres.sum())
        self._fake = None           # (N_f, _DeviceSet, its NativePlans, output buffers) of the last fake set size

    def _plan(self, native, key, compile_fn):
        return native.get(key, compile_fn, (lambda pl: (0,) * S.DS_IO_COUNT) if self.cuda_graph else None)

    def _run(self, native, h):
        native.run(h, (None,) * S.DS_IO_COUNT, torch.cuda.current_stream(self.device).cuda_stream)

    def _fake_buffers(self, Nf):
        if self._fake is None or self._fake[0] != Nf:
            self._fake = None
            z = lambda n, dt: torch.zeros(n, dtype=dt, device=self.device)
            out = dict(cnt_f=z(Nf, torch.int32), realism=z(Nf, torch.float64), nres_fr=z(Nf, torch.int32),
                       cnt_r=z(self.N, torch.int32), own_r=z(self.N, torch.int32), nres_rf=z(self.N, torch.int32))
            self._fake = (Nf, _DeviceSet(Nf, self.D, self.device), _lib.NativePlans((C.c_ubyte * 1024)(), self.device), out)
        return self._fake

    def _score_plan(self, fake_features, realism):
        if realism and not bool((self.radii < self.median).any()):
            raise ValueError('realism: no real radius is below the median of the radii (the reference takes the maximum of an empty set)')
        x = _rows(fake_features, 'fake_features')
        if x.shape[1] != self.D:
            raise ValueError(f'fake_features has {x.shape[1]} features per row, real_features {self.D}')
        _check_rows(x, self.k, 'fake_features')
        x = x.to(self.device)
        Nf, fs, native, out = self._fake_buffers(x.shape[0])
        fs.fill(x)
        del x
        F, R, p = fs.refs, self.real.refs, lambda name: out[name].data_ptr()
        passes = [('kth', F, fs.nres.data_ptr()),
                  ('count', F, R, p('cnt_f'), 0, p('realism') if realism else 0, float(self.median), p('nres_fr')),
                  ('count', R, F, p('cnt_r'), p('own_r'), 0, 0.0, p('nres_rf'))]
        h, pl = self._plan(native, (F.scale, bool(realism)), lambda: compile_plan(passes, self.D, self.k))
        return h, pl, native, fs, out

    @torch.no_grad()
    def score(self, fake_features, realism=False):
        """The reference's dict: precision, recall, density, coverage (numpy float64 scalars) and, with realism=True, realism (float64
        [N_f])."""
        h, _, native, fs, out = self._score_plan(fake_features, realism)
        self._run(native, h)
        cnt_f = out['cnt_f'].cpu().numpy().astype(np.int64)
        cnt_r = out['cnt_r'].cpu().numpy()
        own_r = out['own_r'].cpu().numpy()
        self.last_rescored_pairs = int(fs.nres.sum()) + int(out['nres_fr'].sum()) + int(out['nres_rf'].sum())
        self.fake_radii = fs.rad.cpu().numpy()
        d = dict(precision=(cnt_f > 0).mean(), recall=(cnt_r > 0).mean(), density=(1. / float(self.k)) * cnt_f.mean(),
                 coverage=(own_r > 0).mean())
        if realism:
            d['realism'] = out['realism'].cpu().numpy().copy()
        return d

    def profile_score(self, fake_features, realism=False):
        """One score() with per-op CUDA-event timing: list of (op type, ms)."""
        self.score(fake_features, realism)
        h, pl, native, _, _ = self._score_plan(fake_features, realism)
        lib = native.lib
        _lib.check(lib.ds_unet_set_profiling(h, 1), 'ds_unet_set_profiling')
        self._run(native, h)
        buf = (C.c_float * pl.n_ops)()
        n = lib.ds_unet_get_profile(h, buf, pl.n_ops)
        lib.ds_unet_set_profiling(h, 0)
        return [(lib.ds_unet_op_type(h, i), float(buf[i])) for i in range(n)]


def _device_of(*xs):
    for x in xs:
        if torch.is_tensor(x) and x.is_cuda:
            return x.device
    return None


def compute_prdc(real_features, fake_features, nearest_k, realism=False):
    """sfd-main/prdc.py's compute_prdc: dict of precision, recall, density, coverage (and realism).  Every argument is checked before
    any work on the GPU."""
    k = _check_k(nearest_k)
    device = _device_of(real_features, fake_features)
    real, fake = _rows(real_features, 'real_features'), _rows(fake_features, 'fake_features')
    if real.shape[1] != fake.shape[1]:
        raise ValueError(f'fake_features has {fake.shape[1]} features per row, real_features {real.shape[1]}')
    _check_rows(real, k, 'real_features')
    _check_rows(fake, k, 'fake_features')
    return B200PRDC(real, k, device=device).score(fake, realism=realism)


def compute_nearest_neighbour_distances(input_features, nearest_k):
    """sfd-main/prdc.py's compute_nearest_neighbour_distances: the (nearest_k + 1)-th smallest distance of each row to the set,
    its own distance 0 included (float64 [N])."""
    return B200PRDC(input_features, nearest_k, device=_device_of(input_features)).radii
