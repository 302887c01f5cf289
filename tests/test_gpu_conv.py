"""Unit parity of the two convolution engines (wgmma implicit GEMM / SIMT) against a plain PyTorch fp32
convolution of the same op (cuDNN with TF32 disabled), for every (cin, cout, k, stride, H) family that
occurs in HRNet-W48 (SURVEY.md 8a) plus ragged sizes."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

# (cin, cout, k, stride, H, W, B)
SHAPES = [
    (48, 48, 3, 1, 56, 56, 2),     # 22.5 % of the FLOPs, KCH=16 / SW32
    (96, 96, 3, 1, 28, 28, 2),     # KCH=32 / SW64
    (192, 192, 3, 1, 14, 14, 3),   # KCH=64 / SW128, 2 n-tiles, TH=9 ragged
    (384, 384, 3, 1, 7, 7, 5),     # multi-image tiles (TN=2), odd batch
    (64, 64, 3, 2, 112, 112, 1),   # stem conv2, stride-2 parity views
    (256, 48, 3, 1, 56, 56, 1),    # transition1
    (256, 96, 3, 2, 56, 56, 1),
    (48, 96, 3, 2, 56, 56, 2),     # fuse down-sampling
    (96, 48, 1, 1, 28, 28, 2),     # fuse up-sampling 1x1
    (64, 256, 1, 1, 56, 56, 1),    # bottleneck 1x1
    (1536, 512, 1, 1, 7, 7, 2),
    (512, 2048, 1, 1, 7, 7, 2),    # 16 n-tiles
    (48, 48, 3, 1, 8, 24, 1),      # non-square small map
    (96, 192, 3, 2, 28, 28, 2),    # stride-2 halo variant, KCH=32, two cout tiles
    (48, 48, 3, 2, 16, 24, 3),     # stride-2 halo variant, non-square, whole-image items
    (64, 64, 3, 1, 136, 136, 1),   # W > 128 is not tiled by the wgmma engine -> unsupported, see below
]


def _ref(x, w, b, bn, stride, res, relu):
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        y = F.conv2d(x.permute(0, 3, 1, 2), w, b, stride=stride, padding=w.shape[-1] // 2)
    finally:
        torch.backends.cudnn.allow_tf32 = prev
    if bn is not None:
        y = F.batch_norm(y, bn['mean'], bn['var'], bn['weight'], bn['bias'], False, 0.0, bn['eps'])
    y = y.permute(0, 2, 3, 1)
    if res is not None:
        y = y + res
    return F.relu(y) if relu else y


def _case(cin, cout, k, stride, H, W, B, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, H, W, cin, generator=g)
    w = torch.randn(cout, cin, k, k, generator=g) * (2.0 / (cin * k * k)) ** 0.5
    bn = dict(weight=torch.rand(cout, generator=g) + 0.5, bias=torch.randn(cout, generator=g) * 0.1,
              mean=torch.randn(cout, generator=g) * 0.1, var=torch.rand(cout, generator=g) + 0.5, eps=1e-5)
    Ho, Wo = (H // 2, W // 2) if stride == 2 else (H, W)
    res = torch.randn(B, Ho, Wo, cout, generator=g)
    return x.cuda(), w.cuda(), {k_: (v.cuda() if torch.is_tensor(v) else v) for k_, v in bn.items()}, res.cuda()


def rel(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max())


@pytest.mark.parametrize('shape', SHAPES[:-1])
@pytest.mark.parametrize('engine', [1, 0])
def test_conv_parity_split_mode(shape, engine):
    from shapy_b200 import ops
    cin, cout, k, stride, H, W, B = shape
    x, w, bn, res = _case(*shape)
    ref = _ref(x, w, None, bn, stride, res, True)
    y = ops.conv_test(x, w, bn=bn, stride=stride, res_nhwc=res, relu=True, mode=1, engine=engine)
    assert rel(y, ref) < 2e-5, rel(y, ref)
    # no residual, no relu, conv bias instead of BN (subsample_N / conv_layers.downsample variants)
    bias = torch.randn(cout, device='cuda') * 0.1
    ref = _ref(x, w, bias, None, stride, None, False)
    y = ops.conv_test(x, w, bias=bias, stride=stride, relu=False, mode=1, engine=engine)
    assert rel(y, ref) < 2e-5, rel(y, ref)


@pytest.mark.parametrize('shape', [SHAPES[0], SHAPES[2], SHAPES[4], SHAPES[11]])
def test_conv_fp16_mode(shape):
    """mode 0: fp16 operands, fp32 accumulate; both engines see the same rounded operands."""
    from shapy_b200 import ops
    cin, cout, k, stride, H, W, B = shape
    x, w, bn, res = _case(*shape, seed=1)
    ref = _ref(x, w, None, bn, stride, None, True)
    y0 = ops.conv_test(x, w, bn=bn, stride=stride, relu=True, mode=0, engine=0)
    y1 = ops.conv_test(x, w, bn=bn, stride=stride, relu=True, mode=0, engine=1)
    assert rel(y0, ref) < 5e-3
    assert rel(y0, y1) < 2e-3      # output is rounded to fp16 in this mode


@pytest.mark.parametrize('scale', [300.0, 1.0 / 300.0])
@pytest.mark.parametrize('shape', [SHAPES[0], SHAPES[1], SHAPES[9]])
def test_conv_split_mode_activation_ranges(shape, scale):
    """The hi / lo split keeps ~22 mantissa bits at any magnitude inside fp16's exponent range: activations in the
    hundreds to low thousands (realistic post-BN HRNet ranges) and in the 1e-3 range (where `lo` lives among fp16's
    subnormals and is stored scaled by 2^11) give the same relative error as unit-scale ones.  Values beyond
    65 504 are outside the split representation (DESIGN.md section 3) and are not part of the contract."""
    from shapy_b200 import ops
    cin, cout, k, stride, H, W, B = shape
    x, w, bn, res = _case(*shape, seed=2)
    x, res = x * scale, res * scale
    for b in ('mean', 'bias'):
        bn[b] = bn[b] * scale
    ref = _ref(x, w, None, bn, stride, res, True)
    assert float(ref.abs().max()) < 6.0e4
    y = ops.conv_test(x, w, bn=bn, stride=stride, res_nhwc=res, relu=True, mode=1, engine=0)
    assert rel(y, ref) < 2e-5, rel(y, ref)
    # and elementwise where the reference is not tiny: no element loses more than a few fp32 ulps of the tensor scale
    big = ref.abs() > 1e-2 * ref.abs().max()
    assert float(((y - ref).abs()[big] / ref.abs()[big]).max()) < 2e-3


def test_unsupported_shape_is_reported():
    from shapy_b200 import ops
    x, w, bn, res = _case(*SHAPES[-1])
    with pytest.raises(RuntimeError):
        ops.conv_test(x, w, bn=bn, stride=1, relu=True, mode=1, engine=0)
    y = ops.conv_test(x, w, bn=bn, stride=1, relu=True, mode=1, engine=1)   # the SIMT engine handles it
    assert rel(y, _ref(x, w, None, bn, 1, None, True)) < 2e-5


# the convolution families of the network at the batch sizes BASELINE's configurations run (halo_configure and the
# per-tap tile chooser pick their tiles from the batch): (cin, cout, k, stride, H)
BENCH_SHAPES = [(48, 48, 3, 1, 56), (96, 96, 3, 1, 28), (192, 192, 3, 1, 14), (384, 384, 3, 1, 7), (64, 64, 3, 1, 56),
                (64, 256, 1, 1, 56), (256, 64, 1, 1, 56), (48, 96, 3, 2, 56), (96, 192, 3, 2, 28), (192, 384, 3, 2, 14),
                (192, 48, 1, 1, 14), (2048, 512, 1, 1, 7)]


@pytest.mark.parametrize('shape', BENCH_SHAPES)
def test_conv_split_benchmark_batch(shape):
    """configs[2] launch configurations: B = 64, split-fp16 mode, wgmma engine, with residual."""
    from shapy_b200 import ops
    cin, cout, k, stride, H = shape
    x, w, bn, res = _case(cin, cout, k, stride, H, H, 64, seed=2)
    ref = _ref(x, w, None, bn, stride, res, True)
    y = ops.conv_test(x, w, bn=bn, stride=stride, res_nhwc=res, relu=True, mode=1, engine=0)
    assert rel(y, ref) < 2e-5, rel(y, ref)


@pytest.mark.parametrize('shape', BENCH_SHAPES)
def test_conv_fp16_benchmark_batch(shape):
    """configs[1] launch configurations: B = 32, plain fp16 operands.  Reference: the same operands rounded to fp16
    (BN scale folded into the weights first, as the library does), fp32 accumulation; the library's output is itself
    rounded to fp16, so every element must be within 1 fp16 ulp of the reference."""
    from shapy_b200 import ops
    cin, cout, k, stride, H = shape
    x, w, bn, _ = _case(cin, cout, k, stride, H, H, 32, seed=3)
    s = bn['weight'] / torch.sqrt(bn['var'] + bn['eps'])
    wf = (w * s[:, None, None, None]).half().float()
    shift = bn['bias'] - bn['mean'] * s
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        ref = F.conv2d(x.half().float().permute(0, 3, 1, 2), wf, None, stride=stride, padding=k // 2)
    finally:
        torch.backends.cudnn.allow_tf32 = prev
    ref = F.relu(ref + shift[None, :, None, None]).permute(0, 2, 3, 1)
    y = ops.conv_test(x, w, bn=bn, stride=stride, relu=True, mode=0, engine=0)
    err = (y - ref).abs() / (ref.abs() + 1e-2)
    assert float(err.max()) < 1.2e-3, float(err.max())          # 1 ulp of fp16 = 9.8e-4 relative
    assert float(((y - ref) ** 2).mean().sqrt() / (ref ** 2).mean().sqrt()) < 4e-4
