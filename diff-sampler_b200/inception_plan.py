"""Plan compiler of the FID feature extractor: TensorFlow's `inception-2015-12-05` graph (the detector of fid.py, NVIDIA's
`inception-2015-12-05.pkl`), from weights in torchvision's `Inception3` state-dict layout, lowered onto the native ops.  DESIGN.md 4.10.

  * every BasicConv2d (conv -> BatchNorm(eps 1e-3, running statistics) -> ReLU) is ONE GEMM launch in rows mode: BatchNorm folded into
    the weight and the bias here, the ReLU in the epilogue (ds_gemm_desc.relu);
  * a 1x1 convolution reads the fp16 planes of its input directly (channels past the last whole 64 zero-filled by TMA), a k > 1 one the
    rows of ds_im2col, whose K is (kh, kw, c) dense, padded once at the end to a multiple of 64 -- the weight is packed in that order;
  * each branch writes its columns of the block's concat buffer (ldo = block channels): fp32 for the pools and im2cols of the next block,
    fp16 planes for its 1x1 convolutions, both from one epilogue;
  * the pool branches, the stride-2 max pools of Mixed_6a / Mixed_7a (straight into their concat buffers) and the final 8 x 8 mean are
    ds_pool, the input stage (uint8, TF1 legacy bilinear resize to 299, (v - 128) / 128) is ds_img_input.
Pure host logic — no GPU needed to compile a plan."""
import torch

from . import _cstructs as S
from . import gemm_desc as G
from .plan import F4, H2, PlanBuilder, WeightBlob, io

BN_EPS = 1e-3
RES = 299
FEATURES = 2048

STEM = [  # name, cin, cout, (kh, kw), stride, (ph, pw)
    ('Conv2d_1a_3x3', 3, 32, (3, 3), 2, (0, 0)),
    ('Conv2d_2a_3x3', 32, 32, (3, 3), 1, (0, 0)),
    ('Conv2d_2b_3x3', 32, 64, (3, 3), 1, (1, 1)),
    ('Conv2d_3b_1x1', 64, 80, (1, 1), 1, (0, 0)),
    ('Conv2d_4a_3x3', 80, 192, (3, 3), 1, (0, 0)),
]
# block name, kind, input channels, kind parameter (A: pool features, C: c7)
BLOCKS = [('Mixed_5b', 'A', 192, 32), ('Mixed_5c', 'A', 256, 64), ('Mixed_5d', 'A', 288, 64), ('Mixed_6a', 'B', 288, None),
          ('Mixed_6b', 'C', 768, 128), ('Mixed_6c', 'C', 768, 160), ('Mixed_6d', 'C', 768, 160), ('Mixed_6e', 'C', 768, 192),
          ('Mixed_7a', 'D', 768, None), ('Mixed_7b', 'E', 1280, None), ('Mixed_7c', 'E', 2048, None)]


def _convs(kind, n, cin, p):
    """The BasicConv2d layers of one block: name -> (cin, cout, (kh, kw), stride, (ph, pw))."""
    one = lambda ci, co: (ci, co, (1, 1), 1, (0, 0))
    if kind == 'A':
        L = {'branch1x1': one(cin, 64), 'branch5x5_1': one(cin, 48), 'branch5x5_2': (48, 64, (5, 5), 1, (2, 2)),
             'branch3x3dbl_1': one(cin, 64), 'branch3x3dbl_2': (64, 96, (3, 3), 1, (1, 1)), 'branch3x3dbl_3': (96, 96, (3, 3), 1, (1, 1)),
             'branch_pool': one(cin, p)}
    elif kind == 'B':
        L = {'branch3x3': (cin, 384, (3, 3), 2, (0, 0)), 'branch3x3dbl_1': one(cin, 64),
             'branch3x3dbl_2': (64, 96, (3, 3), 1, (1, 1)), 'branch3x3dbl_3': (96, 96, (3, 3), 2, (0, 0))}
    elif kind == 'C':
        row = lambda ci, co: (ci, co, (1, 7), 1, (0, 3))
        col = lambda ci, co: (ci, co, (7, 1), 1, (3, 0))
        L = {'branch1x1': one(cin, 192), 'branch7x7_1': one(cin, p), 'branch7x7_2': row(p, p), 'branch7x7_3': col(p, 192),
             'branch7x7dbl_1': one(cin, p), 'branch7x7dbl_2': col(p, p), 'branch7x7dbl_3': row(p, p), 'branch7x7dbl_4': col(p, p),
             'branch7x7dbl_5': row(p, 192), 'branch_pool': one(cin, 192)}
    elif kind == 'D':
        L = {'branch3x3_1': one(cin, 192), 'branch3x3_2': (192, 320, (3, 3), 2, (0, 0)), 'branch7x7x3_1': one(cin, 192),
             'branch7x7x3_2': (192, 192, (1, 7), 1, (0, 3)), 'branch7x7x3_3': (192, 192, (7, 1), 1, (3, 0)),
             'branch7x7x3_4': (192, 192, (3, 3), 2, (0, 0))}
    else:
        L = {'branch1x1': one(cin, 320), 'branch3x3_1': one(cin, 384), 'branch3x3_2a': (384, 384, (1, 3), 1, (0, 1)),
             'branch3x3_2b': (384, 384, (3, 1), 1, (1, 0)), 'branch3x3dbl_1': one(cin, 448), 'branch3x3dbl_2': (448, 384, (3, 3), 1, (1, 1)),
             'branch3x3dbl_3a': (384, 384, (1, 3), 1, (0, 1)), 'branch3x3dbl_3b': (384, 384, (3, 1), 1, (1, 0)), 'branch_pool': one(cin, 192)}
    return {f'{n}.{k}': v for k, v in L.items()}


def layers():
    """Every BasicConv2d of the net in state-dict order: name -> (cin, cout, (kh, kw), stride, (ph, pw))."""
    out = {name: (ci, co, k, s, p) for name, ci, co, k, s, p in STEM}
    for n, kind, cin, p in BLOCKS:
        out.update(_convs(kind, n, cin, p))
    return out


def required_keys():
    """The state-dict keys the extractor reads (conv weight and the four BatchNorm tensors of every BasicConv2d)."""
    return [f'{n}.{t}' for n in layers() for t in ('conv.weight', 'bn.weight', 'bn.bias', 'bn.running_mean', 'bn.running_var')]


def fold_bn(sd, name):
    """conv (no bias) -> BatchNorm(eps 1e-3, running statistics) of BasicConv2d `name` as one convolution: (weight [cout, kh*kw*cin]
    with K ordered (kh, kw, c), bias [cout]), float64."""
    w = sd[name + '.conv.weight'].double()
    a = sd[name + '.bn.weight'].double() / torch.sqrt(sd[name + '.bn.running_var'].double() + BN_EPS)
    b = sd[name + '.bn.bias'].double() - sd[name + '.bn.running_mean'].double() * a
    return (w * a[:, None, None, None]).permute(0, 2, 3, 1).reshape(w.shape[0], -1), b


def pack_inception_weights(sd):
    """The weight blob: per BasicConv2d `name`, the folded weight as fp16 hi/lo planes [2][cout_pad][K64] (`name`:w) and the fp32
    bias (`name`:b)."""
    wb = WeightBlob()
    for name in layers():
        w, b = fold_bn(sd, name)
        wb.add_gemm(name, w.float(), bias=b.float())
    return wb


def _out(n, k, s, p):
    return (n + 2 * p - k) // s + 1


def compile_inception_plan(wb, B, H, W, npass=3, strides=None):
    """Features of B uint8 images [B][3][H][W] (io X; element strides `strides` = (sn, sc, sy, sx), default contiguous NCHW) into io D
    [B][2048] fp32."""
    sn, sc, sy, sx = strides or (3 * H * W, H * W, W, 1)
    pb = PlanBuilder(wb, B, npass)
    Wt = wb.ref
    npl = 2 if npass == 3 else 1            # fp16 planes of every GEMM operand the plan writes: the lo plane only for fp16x3
    L = layers()

    pb.need('img', B * RES * RES * 3 * F4)
    pb.emit(lambda R: S.ImgInputDesc(src=io(S.DS_IO_X), out=R('img'), sn=sn, sc=sc, sy=sy, sx=sx, B=B, C=3, H=H, W=W, Ho=RES, Wo=RES))

    def conv(name, src, h, w, dst, pitch, c0=0, dst16=None, src16=None):
        """BasicConv2d `name` over the h x w input (fp32 `src`, dense; or, 1x1, its fp16 planes `src16`) into channels c0.. of the
        fp32 buffer `dst` (and its fp16 planes `dst16`) of channel pitch `pitch`.  Returns the output size."""
        cin, cout, (kh, kw), s, (ph, pw) = L[name]
        ho, wo = _out(h, kh, s, ph), _out(w, kw, s, pw)
        M = B * ho * wo
        K64 = -(-(kh * kw * cin) // 64) * 64
        if src16 is not None:
            assert (kh, kw, s) == (1, 1, 1)
            a, a_pitch, a_kv = src16, cin, cin
        else:
            pb.need('cols', npl * M * K64 * H2)
            pb.emit(lambda R: S.Im2colDesc(src=R(src), out=R('cols'), B=B, H=h, W=w, C=cin, src_pitch=cin, src_c0=0, kh=kh, kw=kw,
                                           sh=s, sw=s, ph=ph, pw=pw, K64=K64, nplanes=npl))
            a, a_pitch, a_kv = 'cols', K64, None
        pb.need(dst, M * pitch * F4)
        if dst16:
            pb.need(dst16, npl * M * pitch * H2)
        pb.emit(lambda R: G.rows_gemm(R(a), M, a_pitch, 1, Wt(name + ':w'), G.padded_rows(cout), K64, 1, K64, num_z=1, m_valid=M,
                                      n_valid=cout, npass=npass, a_planes=npl, out_f32=R(dst, 4 * c0), ldo=pitch, bias_n=Wt(name + ':b'),
                                      out_h16=R(dst16, 2 * c0) if dst16 else 0, o_plane=M * pitch if dst16 and npl == 2 else 0,
                                      a_k_valid=a_kv, relu=1)[0])
        return ho, wo

    def pool(src, h, w, c, mode, k, s, p, dst=None, dst16=None, pitch=None, c0=0, src_pitch=None):
        ho, wo = _out(h, k, s, p), _out(w, k, s, p)
        pitch = pitch or c
        if dst:
            pb.need(dst, B * ho * wo * pitch * F4)
        if dst16:
            pb.need(dst16, npl * B * ho * wo * pitch * H2)
        pb.emit(lambda R: S.PoolDesc(src=R(src), out_f32=R(dst) if dst else 0, out_h16=R(dst16) if dst16 else 0,
                                     B=B, H=h, W=w, C=c, src_pitch=src_pitch or c, src_c0=0, out_pitch=pitch, out_c0=c0, k=k, stride=s,
                                     pad=p, mode=mode, nplanes=npl))
        return ho, wo

    # ---- stem: 299 -> 149 -> 147 -> 147 -> 73 -> 73 -> 71 -> 35
    h, w = conv('Conv2d_1a_3x3', 'img', RES, RES, 'a', 32)
    h, w = conv('Conv2d_2a_3x3', 'a', h, w, 'b', 32)
    h, w = conv('Conv2d_2b_3x3', 'b', h, w, 'a', 64)
    h, w = pool('a', h, w, 64, S.DS_POOL_MAX, 3, 2, 0, dst16='p16')
    h, w = conv('Conv2d_3b_1x1', None, h, w, 'b', 80, src16='p16')
    h, w = conv('Conv2d_4a_3x3', 'b', h, w, 'a', 192)
    h, w = pool('a', h, w, 192, S.DS_POOL_MAX, 3, 2, 0, dst='x', dst16='x16')

    # ---- the Mixed blocks: input (x, x16), output (y, y16), then swapped
    cur, cur16, nxt, nxt16 = 'x', 'x16', 'y', 'y16'
    for n, kind, cin, p in BLOCKS:
        pb.tag += 1
        last = n == BLOCKS[-1][0]
        o16 = None if last else nxt16
        if kind == 'A':
            cout = 224 + p
            conv(n + '.branch1x1', None, h, w, nxt, cout, 0, o16, src16=cur16)
            conv(n + '.branch5x5_1', None, h, w, 't1', 48, src16=cur16)
            conv(n + '.branch5x5_2', 't1', h, w, nxt, cout, 64, o16)
            conv(n + '.branch3x3dbl_1', None, h, w, 't1', 64, src16=cur16)
            conv(n + '.branch3x3dbl_2', 't1', h, w, 't2', 96)
            conv(n + '.branch3x3dbl_3', 't2', h, w, nxt, cout, 128, o16)
            pool(cur, h, w, cin, S.DS_POOL_AVG, 3, 1, 1, dst16='pool16')
            conv(n + '.branch_pool', None, h, w, nxt, cout, 224, o16, src16='pool16')
        elif kind == 'B':
            cout = 768
            conv(n + '.branch3x3', cur, h, w, nxt, cout, 0, o16)
            conv(n + '.branch3x3dbl_1', None, h, w, 't1', 64, src16=cur16)
            conv(n + '.branch3x3dbl_2', 't1', h, w, 't2', 96)
            conv(n + '.branch3x3dbl_3', 't2', h, w, nxt, cout, 384, o16)
            h, w = pool(cur, h, w, cin, S.DS_POOL_MAX, 3, 2, 0, dst=nxt, dst16=o16, pitch=cout, c0=480)
        elif kind == 'C':
            cout = 768
            conv(n + '.branch1x1', None, h, w, nxt, cout, 0, o16, src16=cur16)
            conv(n + '.branch7x7_1', None, h, w, 't1', p, src16=cur16)
            conv(n + '.branch7x7_2', 't1', h, w, 't2', p)
            conv(n + '.branch7x7_3', 't2', h, w, nxt, cout, 192, o16)
            conv(n + '.branch7x7dbl_1', None, h, w, 't1', p, src16=cur16)
            conv(n + '.branch7x7dbl_2', 't1', h, w, 't2', p)
            conv(n + '.branch7x7dbl_3', 't2', h, w, 't1', p)
            conv(n + '.branch7x7dbl_4', 't1', h, w, 't2', p)
            conv(n + '.branch7x7dbl_5', 't2', h, w, nxt, cout, 384, o16)
            pool(cur, h, w, cin, S.DS_POOL_AVG, 3, 1, 1, dst16='pool16')
            conv(n + '.branch_pool', None, h, w, nxt, cout, 576, o16, src16='pool16')
        elif kind == 'D':
            cout = 1280
            conv(n + '.branch3x3_1', None, h, w, 't1', 192, src16=cur16)
            conv(n + '.branch3x3_2', 't1', h, w, nxt, cout, 0, o16)
            conv(n + '.branch7x7x3_1', None, h, w, 't1', 192, src16=cur16)
            conv(n + '.branch7x7x3_2', 't1', h, w, 't2', 192)
            conv(n + '.branch7x7x3_3', 't2', h, w, 't1', 192)
            conv(n + '.branch7x7x3_4', 't1', h, w, nxt, cout, 320, o16)
            h, w = pool(cur, h, w, cin, S.DS_POOL_MAX, 3, 2, 0, dst=nxt, dst16=o16, pitch=cout, c0=512)
        else:
            cout = 2048
            conv(n + '.branch1x1', None, h, w, nxt, cout, 0, o16, src16=cur16)
            conv(n + '.branch3x3_1', None, h, w, 't1', 384, src16=cur16)
            conv(n + '.branch3x3_2a', 't1', h, w, nxt, cout, 320, o16)
            conv(n + '.branch3x3_2b', 't1', h, w, nxt, cout, 704, o16)
            conv(n + '.branch3x3dbl_1', None, h, w, 't1', 448, src16=cur16)
            conv(n + '.branch3x3dbl_2', 't1', h, w, 't2', 384)
            conv(n + '.branch3x3dbl_3a', 't2', h, w, nxt, cout, 1088, o16)
            conv(n + '.branch3x3dbl_3b', 't2', h, w, nxt, cout, 1472, o16)
            # the graph's own pools: Mixed_7c's is a max pool, every other one averages without the padding
            pool(cur, h, w, cin, S.DS_POOL_MAX if last else S.DS_POOL_AVG, 3, 1, 1, dst16='pool16')
            conv(n + '.branch_pool', None, h, w, nxt, cout, 1856, o16, src16='pool16')
        cur, cur16, nxt, nxt16 = nxt, nxt16, cur, cur16
    assert (h, w, cout) == (8, 8, FEATURES)

    # ---- pool3: the mean over the 8 x 8 map
    pb.emit(lambda R: S.PoolDesc(src=R(cur), out_f32=io(S.DS_IO_D), B=B, H=h, W=w, C=FEATURES, src_pitch=FEATURES, out_pitch=FEATURES,
                                 mode=S.DS_POOL_MEAN, nplanes=npl))
    return pb.finish(B=B, H=H, W=W, npass=npass, strides=(sn, sc, sy, sx))
