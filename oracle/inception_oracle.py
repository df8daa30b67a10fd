"""ORACLE — test infrastructure, not product code.

Float64 functional restatement of the FID feature extractor: TensorFlow's `inception-2015-12-05` graph (NVIDIA's
`inception-2015-12-05.pkl` is a direct PyTorch translation of it; pytorch-fid's `pt_inception-2015-12-05` holds the same weights in
torchvision's `Inception3` layout, which is the layout read here).

    features(images_u8, sd) -> [B, 2048] float64

  * input stage (`input_stage`): uint8 -> float, TF1 legacy ResizeBilinear to 299 x 299 (source (i H / 299, j W / 299), neighbours
    floor and floor + 1 clamped to the last row / column, no half-pixel centres, no antialiasing), then (v - 128) / 128;
  * body: torchvision's Inception3 wiring, every BasicConv2d = conv (no bias) -> BatchNorm (eps 1e-3, running statistics) -> ReLU;
  * tf_quirks (the graph's own pools, as pytorch-fid patches them): the pool branch of Mixed_5b..5d, 6b..6e and 7b averages 3 x 3
    stride 1 pad 1 WITHOUT the padding in the count, that of Mixed_7c is a 3 x 3 stride 1 pad 1 MAX pool.  tf_quirks=False: torchvision's
    own pools (average including the padding), for pinning the wiring to torchvision itself;
  * output: the mean over the 8 x 8 map of Mixed_7c.
"""
import torch
import torch.nn.functional as F

BN_EPS = 1e-3


def resize_tf_legacy(x, size=299):
    """x: [B, C, H, W] float64 -> [B, C, size, size], TF1 ResizeBilinear(align_corners=False, half_pixel_centers=False)."""
    B, C, H, W = x.shape

    def axis(n):
        f = torch.arange(size, dtype=torch.float64, device=x.device) * n / size
        i0 = f.floor().long()
        return i0, (i0 + 1).clamp(max=n - 1), f - i0
    y0, y1, dy = axis(H)
    x0, x1, dx = axis(W)
    top = x[:, :, y0][..., x0] + (x[:, :, y0][..., x1] - x[:, :, y0][..., x0]) * dx
    bot = x[:, :, y1][..., x0] + (x[:, :, y1][..., x1] - x[:, :, y1][..., x0]) * dx
    return top + (bot - top) * dy[:, None]


def input_stage(images_u8):
    """uint8 [B, 3, H, W] (any strides) -> the network input [B, 3, 299, 299] float64."""
    x = images_u8.to(torch.float64)
    return (resize_tf_legacy(x) - 128.0) / 128.0


def basic_conv(x, sd, name, stride=1, padding=0):
    w = sd[name + '.conv.weight'].double()
    y = F.conv2d(x, w, stride=stride, padding=padding)
    g, b = sd[name + '.bn.weight'].double(), sd[name + '.bn.bias'].double()
    m, v = sd[name + '.bn.running_mean'].double(), sd[name + '.bn.running_var'].double()
    y = (y - m[:, None, None]) / torch.sqrt(v[:, None, None] + BN_EPS) * g[:, None, None] + b[:, None, None]
    return F.relu(y)


def _avg(x, quirks):
    return F.avg_pool2d(x, 3, 1, 1, count_include_pad=not quirks)


def block_a(x, sd, n, quirks):
    b1 = basic_conv(x, sd, n + '.branch1x1')
    b5 = basic_conv(basic_conv(x, sd, n + '.branch5x5_1'), sd, n + '.branch5x5_2', padding=2)
    b3 = basic_conv(x, sd, n + '.branch3x3dbl_1')
    b3 = basic_conv(basic_conv(b3, sd, n + '.branch3x3dbl_2', padding=1), sd, n + '.branch3x3dbl_3', padding=1)
    bp = basic_conv(_avg(x, quirks), sd, n + '.branch_pool')
    return torch.cat([b1, b5, b3, bp], 1)


def block_b(x, sd, n):
    b3 = basic_conv(x, sd, n + '.branch3x3', stride=2)
    bd = basic_conv(x, sd, n + '.branch3x3dbl_1')
    bd = basic_conv(basic_conv(bd, sd, n + '.branch3x3dbl_2', padding=1), sd, n + '.branch3x3dbl_3', stride=2)
    return torch.cat([b3, bd, F.max_pool2d(x, 3, 2)], 1)


def block_c(x, sd, n, quirks):
    b1 = basic_conv(x, sd, n + '.branch1x1')
    b7 = basic_conv(x, sd, n + '.branch7x7_1')
    b7 = basic_conv(b7, sd, n + '.branch7x7_2', padding=(0, 3))
    b7 = basic_conv(b7, sd, n + '.branch7x7_3', padding=(3, 0))
    bd = basic_conv(x, sd, n + '.branch7x7dbl_1')
    for k, p in ((2, (3, 0)), (3, (0, 3)), (4, (3, 0)), (5, (0, 3))):
        bd = basic_conv(bd, sd, f'{n}.branch7x7dbl_{k}', padding=p)
    bp = basic_conv(_avg(x, quirks), sd, n + '.branch_pool')
    return torch.cat([b1, b7, bd, bp], 1)


def block_d(x, sd, n):
    b3 = basic_conv(basic_conv(x, sd, n + '.branch3x3_1'), sd, n + '.branch3x3_2', stride=2)
    b7 = basic_conv(x, sd, n + '.branch7x7x3_1')
    b7 = basic_conv(b7, sd, n + '.branch7x7x3_2', padding=(0, 3))
    b7 = basic_conv(b7, sd, n + '.branch7x7x3_3', padding=(3, 0))
    b7 = basic_conv(b7, sd, n + '.branch7x7x3_4', stride=2)
    return torch.cat([b3, b7, F.max_pool2d(x, 3, 2)], 1)


def block_e(x, sd, n, quirks, pool_max=False):
    b1 = basic_conv(x, sd, n + '.branch1x1')
    b3 = basic_conv(x, sd, n + '.branch3x3_1')
    b3 = torch.cat([basic_conv(b3, sd, n + '.branch3x3_2a', padding=(0, 1)), basic_conv(b3, sd, n + '.branch3x3_2b', padding=(1, 0))], 1)
    bd = basic_conv(basic_conv(x, sd, n + '.branch3x3dbl_1'), sd, n + '.branch3x3dbl_2', padding=1)
    bd = torch.cat([basic_conv(bd, sd, n + '.branch3x3dbl_3a', padding=(0, 1)), basic_conv(bd, sd, n + '.branch3x3dbl_3b', padding=(1, 0))], 1)
    p = F.max_pool2d(x, 3, 1, 1) if (quirks and pool_max) else _avg(x, quirks)
    bp = basic_conv(p, sd, n + '.branch_pool')
    return torch.cat([b1, b3, bd, bp], 1)


def body(x, sd, tf_quirks=True):
    """The network input [B, 3, 299, 299] -> the Mixed_7c map [B, 2048, 8, 8], float64."""
    x = basic_conv(x, sd, 'Conv2d_1a_3x3', stride=2)
    x = basic_conv(x, sd, 'Conv2d_2a_3x3')
    x = basic_conv(x, sd, 'Conv2d_2b_3x3', padding=1)
    x = F.max_pool2d(x, 3, 2)
    x = basic_conv(x, sd, 'Conv2d_3b_1x1')
    x = basic_conv(x, sd, 'Conv2d_4a_3x3')
    x = F.max_pool2d(x, 3, 2)
    for n in ('Mixed_5b', 'Mixed_5c', 'Mixed_5d'):
        x = block_a(x, sd, n, tf_quirks)
    x = block_b(x, sd, 'Mixed_6a')
    for n in ('Mixed_6b', 'Mixed_6c', 'Mixed_6d', 'Mixed_6e'):
        x = block_c(x, sd, n, tf_quirks)
    x = block_d(x, sd, 'Mixed_7a')
    x = block_e(x, sd, 'Mixed_7b', tf_quirks)
    return block_e(x, sd, 'Mixed_7c', tf_quirks, pool_max=True)


def features(images_u8, sd, tf_quirks=True):
    """uint8 images [B, 3, H, W] -> pool3 features [B, 2048] float64."""
    return body(input_stage(images_u8), sd, tf_quirks).mean(dim=(2, 3))


def make_state_dict(seed=0, calib_sizes=(32, 64, 256, 299)):
    """torchvision Inception3 weights (its own random init, seeded) with BatchNorm running statistics calibrated by one train-mode pass
    (momentum=None: the statistics of that one batch) over seeded random uint8 images, two at each size of `calib_sizes`, through the
    input stage, so activations stay moderate through all 94 layers at every input size the tests use.
    Returns the float32 state dict without fc.* / AuxLogits.* / num_batches_tracked."""
    import torchvision
    torch.manual_seed(seed)
    m = torchvision.models.inception_v3(weights=None, aux_logits=False, init_weights=True, transform_input=False)
    for mod in m.modules():
        if isinstance(mod, torch.nn.BatchNorm2d):
            mod.momentum = None
            mod.reset_running_stats()
    g = torch.Generator().manual_seed(seed + 1)
    x = torch.cat([input_stage(torch.randint(0, 256, (2, 3, r, r), generator=g, dtype=torch.uint8)) for r in calib_sizes])
    m.train()
    with torch.no_grad():
        m(x.float())
    return {k: v.detach().clone() for k, v in m.state_dict().items()
            if not (k.startswith('fc.') or k.startswith('AuxLogits.') or k.endswith('num_batches_tracked'))}
