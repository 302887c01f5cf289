"""Every (data path, cout tile NT, consumer schedule) the wgmma convolution engine admits, forced one at a time through
conv_test and checked three ways: the plan it reports is the one forced, the output is within the float64 oracle's
per-element bound (tests/conv_oracle.py), and the outputs agree bit for bit where the arithmetic says they must.

NT and the schedule change neither the k-order nor the epilogue arithmetic, so within one precision mode and one data
path every (NT, schedule) gives the same bits; the weight-resident path issues the halo path's k16 steps in the same
order, so it equals the halo path; with cin <= 64 (one channel block) the per-tap and halo orders coincide too.  An
element's k16 order depends on the path alone, so a batch's first images give the same bits alone as in a larger
batch.  Each shape runs at a small batch (few tiles: for most candidates at most one per CTA) and a large one that
gives every candidate at least two tiles per CTA (asserted from the planner's tiling): the staging box reused,
residual loads under a pending store, the ring wrapped, ping-pong hand-offs.

Run with -s to see one line per candidate with its error-to-bound ratio."""
import math

import pytest
import torch

import conv_oracle as co
from test_gpu_conv import _case

pytestmark = pytest.mark.gpu

PER_TAP, HALO, RESIDENT = 2, 3, 4          # conv_test engine digits (ops.ConvPlan)
COOP, PINGPONG = 1, 2
NTS = (128, 96, 64, 48, 32, 16)            # cout tiles with a kernel instantiation
NAMES = {PER_TAP: 'per-tap', HALO: 'halo', RESIDENT: 'resident', COOP: 'coop', PINGPONG: 'pp'}

# (cin, cout, k, stride, H, W, B small, B large), each chosen for an edge
SHAPES = [
    (48, 48, 3, 1, 56, 56, 1, 10),         # resident, halo and per-tap at NT 48 and 16; CW 16 with three column boxes
    (64, 64, 3, 1, 56, 56, 1, 10),         # resident at NT 64 in fp16 (the split weights of cin 64 do not fit)
    (32, 64, 3, 1, 28, 28, 2, 38),         # resident at NT 64 in split mode too, with two 16-channel slices
    (16, 64, 3, 1, 28, 28, 2, 38),         # resident with one slice
    (96, 96, 3, 1, 28, 28, 2, 38),         # halo, two channel blocks; NT 96 has CW 32 with three boxes
    (192, 192, 3, 1, 14, 14, 4, 66),       # three channel blocks on the two-slot halo ring; per-tap TH 9 ragged
    (384, 384, 3, 1, 7, 7, 3, 175),        # per-tap multi-image tiles (TN 2) at odd B: rows past N
    (192, 384, 3, 2, 14, 14, 3, 175),      # the concat layer: stride-2 parity maps
    (64, 256, 1, 1, 56, 56, 1, 5),         # NT 128 (fp16) and 64
    (384, 48, 1, 1, 7, 7, 2, 527),         # the NT 16 layer the network runs
    (384, 96, 1, 1, 7, 7, 2, 527),         # the NT 32 layer
    (1536, 2048, 1, 1, 7, 7, 1, 33),       # NT 128 with 24 k-blocks
    (80, 80, 3, 1, 20, 20, 2, 16),         # two k-blocks, the last one k16 step long; only NT 16 divides 80
    (144, 160, 3, 2, 28, 28, 2, 27),       # three k-blocks, NT 32 or 16
    (16, 112, 3, 1, 13, 24, 2, 13),        # a single k16 step, NT 16 only, a ragged band
    (64, 64, 1, 1, 8, 256, 1, 17),         # output W 256: two width tiles of 128
    (48, 96, 3, 2, 8, 256, 1, 66),         # stride 2, output W 128
    (384, 384, 3, 1, 2, 3, 7, 1829),       # the smallest map (64 x 96 input): B 7 in one tile
]
# shapes also read through an input view with poisoned surplus channels
IN_VIEW_SHAPES = {(48, 48, 3, 1, 56, 56), (80, 80, 3, 1, 20, 20), (144, 160, 3, 2, 28, 28), (16, 112, 3, 1, 13, 24)}
POISON = 30000.0           # finite: split_store would clamp a NaN into range
# (shape[:6], mode, path, nt, schedule) -> the exact error of a candidate the engine cannot plan: the split-mode
# weight set of a 64 -> 64 3x3 layer (144 KB) with its halo slots and staging box exceeds 227 KB at any width.
_RES64 = 'wgmma_plan_create: the weight-resident path does not fit shared memory (cin 64 cout 64, {} B)'
INFEASIBLE = {
    ((64, 64, 3, 1, 56, 56), 1, RESIDENT, 64, COOP): _RES64.format(308296),
    ((64, 64, 3, 1, 56, 56), 1, RESIDENT, 64, PINGPONG): _RES64.format(341064),
}


def _sid(s):
    cin, cout, k, st, H, W, bs, bl = s
    return f'{cin}-{cout}-k{k}s{st}-{H}x{W}-b{bs}-{bl}'


def candidates(cin, cout, k, stride, Wo, mode):
    paths = [PER_TAP]
    if k == 3 and stride == 1 and Wo + 2 <= 128:
        paths.append(HALO)
        if cin <= 64 and cout in (48, 64):
            paths.append(RESIDENT)
    out = []
    for path in paths:
        for nt in NTS:
            if cout % nt or (mode and nt > 96) or (path == RESIDENT and nt != cout):
                continue
            out.append((path, nt, COOP))
            if nt <= (64 if mode else 128):          # the ping-pong accumulators fit
                out.append((path, nt, PINGPONG))
    return out


def work_items(cin, cout, k, stride, H, W, B, cand):
    """Tiles of a launch as wgmma_plan_create lays them out: M tiles x cout tiles."""
    path, nt, _ = cand
    Ho, Wo = H // stride, W // stride
    if path == PER_TAP:
        TW = min(Wo, 128)
        TH = max(1, min(Ho, 128 // TW))
        TN = max(1, min(B, 128 // (TW * TH))) if (TW, TH) == (Wo, Ho) else 1
        m = -(-Wo // TW) * -(-Ho // TH) * -(-B // TN)
    else:                                    # halo bands of balanced height on the padded grid
        per = 128 // (Wo + 2)
        th = -(-Ho // -(-Ho // per))
        m = -(-Ho // th) * B
    return m * (cout // nt)


def engine(cand):
    path, nt, sched = cand
    return path + 10 * sched + 100 * nt


def kernel_of(mode, cand):
    """The conv_wgmma_kernel<SPLIT, NT, HALO, PP, RES> instantiation a candidate runs."""
    path, nt, sched = cand
    return (bool(mode), nt, path != PER_TAP, sched == PINGPONG, path == RESIDENT)


def cw(nt):
    return 64 if nt % 64 == 0 else (32 if nt % 32 == 0 else 16)


def _run(x, w, cand, **kw):
    from shapy_b200 import ops
    y, plan = ops.conv_test(x, w, engine=engine(cand), report=True, **kw)
    assert (plan.path, plan.nt, plan.schedule) == cand, (plan, cand)
    return y


def _log(shape, mode, cand, what, r):
    print(f'[tiles] {shape} mode {mode} {NAMES[cand[0]]} NT {cand[1]} {NAMES[cand[2]]} {what}: ratio {r:.3g}')


def _plannable(shape, mode, cands, run):
    """Runs run(cand) for every candidate; a plan failure must be pinned in INFEASIBLE with its exact message."""
    out, failed = {}, set()
    for c in cands:
        try:
            out[c] = run(c)
        except RuntimeError as e:
            key = (shape, mode) + c
            assert key in INFEASIBLE and INFEASIBLE[key] in str(e), (key, str(e))
            failed.add(key)
    pinned = {k for k in INFEASIBLE if k[:2] == (shape, mode) and k[2:] in cands}
    assert failed == pinned, ('pinned candidates planned after all', pinned - failed)
    return out


@pytest.mark.parametrize('mode', [1, 0])
@pytest.mark.parametrize('shape', SHAPES, ids=_sid)
def test_every_tile_and_schedule(shape, mode):
    cin, cout, k, s, H, W, Bs, Bl = shape
    x, w, bn, res = _case(cin, cout, k, s, H, W, Bl, seed=20)
    kw = dict(bn=bn, stride=s, relu=True, mode=mode)
    ref = co.reference(x, w, bn=bn, stride=s, res=res, relu=True, mode=mode)
    cands = candidates(cin, cout, k, s, W // s, mode)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert min(work_items(cin, cout, k, s, H, W, Bl, c) for c in cands) >= 2 * sms

    def run(c):
        y = _run(x, w, c, res_nhwc=res, **kw)
        r = co.ratio(y, ref)
        _log(shape[:6], mode, c, f'B {Bl}', r)
        assert r <= 1.0, (c, co.worst(y, ref))
        y_s = _run(x[:Bs], w, c, res_nhwc=res[:Bs], **kw)
        assert torch.equal(y_s, y[:Bs]), c
        if shape[:6] in IN_VIEW_SHAPES:         # channels 16 .. 16 + cin of cin + 48, the rest poison
            xv = torch.full((Bs, H, W, cin + 48), POISON, device=x.device)
            xv[..., 16:16 + cin] = x[:Bs]
            assert torch.equal(_run(xv, w, c, res_nhwc=res[:Bs], in_view=(cin + 48, 16), **kw), y_s), c
        return y
    outs = _plannable(shape[:6], mode, cands, run)
    assert outs
    for path in (PER_TAP, HALO, RESIDENT):
        ys = [y for c, y in outs.items() if c[0] == path]
        for y in ys[1:]:
            assert torch.equal(y, ys[0]), path
    first = {c[0]: y for c, y in outs.items()}
    if RESIDENT in first:
        assert torch.equal(first[RESIDENT], first[HALO])
    if cin <= 64:
        for y in first.values():
            assert torch.equal(y, next(iter(first.values())))


# epilogue variants: (residual, ReLU, conv bias in place of BN)
VARIANTS = [(False, True, False), (True, False, False), (False, False, True)]


@pytest.mark.parametrize('mode', [1, 0])
@pytest.mark.parametrize('shape', SHAPES, ids=_sid)
def test_epilogue_variants(shape, mode):
    """Each variant on, per path, the widest NT of each column-box width, in both schedules."""
    cin, cout, k, s, H, W, _, Bl = shape
    x, w, bn, res = _case(cin, cout, k, s, H, W, Bl, seed=21)
    bias = torch.randn(cout, device='cuda') * 0.1
    cands = candidates(cin, cout, k, s, W // s, mode)
    widest = {}
    for c in cands:
        widest.setdefault((c[0], cw(c[1])), c[1])
    cands = [c for c in cands if widest[(c[0], cw(c[1]))] == c[1]]
    for with_res, relu, with_bias in VARIANTS:
        kw = dict(bias=bias if with_bias else None, bn=None if with_bias else bn, stride=s,
                  res=res if with_res else None, relu=relu, mode=mode)
        ref = co.reference(x, w, **kw)
        kw['res_nhwc'] = kw.pop('res')

        def run(c):
            y = _run(x, w, c, **kw)
            r = co.ratio(y, ref)
            _log(shape[:6], mode, c, f'res {with_res} relu {relu} bias {with_bias}', r)
            assert r <= 1.0, (c, co.worst(y, ref))
            return y
        outs = _plannable(shape[:6], mode, cands, run)
        for path in (PER_TAP, HALO, RESIDENT):
            ys = [y for c, y in outs.items() if c[0] == path]
            for y in ys[1:]:
                assert torch.equal(y, ys[0]), path


# the concat layer writes slices of the 1536-channel tensor; 1144 is a multiple of 8 but not of 16
@pytest.mark.parametrize('coff', [0, 384, 768, 1144])
@pytest.mark.parametrize('mode', [1, 0])
def test_concat_output_views(mode, coff):
    cin, cout, k, s, H, W, B = 192, 384, 3, 2, 14, 14, 5
    x, w, bn, _ = _case(cin, cout, k, s, H, W, B, seed=22)
    kw = dict(bn=bn, stride=s, relu=True, mode=mode)
    ref = co.reference(x, w, **kw)
    dense = None

    def run(c):
        nonlocal dense
        y = _run(x, w, c, out_view=(1536, coff), **kw)
        assert y.shape == (B + 1, H // 2, W // 2, 1536)
        sl = y[:B, ..., coff:coff + cout]
        assert not sl.isnan().any(), c
        r = co.ratio(sl, ref)
        _log((cin, cout, k, s, H, W), mode, c, f'out_view (1536, {coff})', r)
        assert r <= 1.0, (c, co.worst(sl, ref))
        outside = torch.ones_like(y, dtype=torch.bool)
        outside[:B, ..., coff:coff + cout] = False
        assert y[outside].isnan().all(), c          # the other channels and the guard image are untouched
        if dense is None:
            dense = _run(x, w, c, **kw)
        assert torch.equal(sl, dense), c
        return y
    _plannable((cin, cout, k, s, H, W), mode, candidates(cin, cout, k, s, W // s, mode), run)


def test_reached_kernels():
    """The candidates above reach every one of the 50 kernel instantiations."""
    reached = set()
    for shape in SHAPES:
        cin, cout, k, s, H, W, _, _ = shape
        for mode in (1, 0):
            reached |= {kernel_of(mode, c) for c in candidates(cin, cout, k, s, W // s, mode)
                        if (shape[:6], mode) + c not in INFEASIBLE}
    every = set()
    for split in (True, False):
        for nt in NTS:
            if split and nt > 96:
                continue
            for halo in (False, True):
                for pp in (False, True):
                    if pp and nt > (64 if split else 128):
                        continue
                    every.add((split, nt, halo, pp, False))
                    if halo and nt in (48, 64):
                        every.add((split, nt, halo, pp, True))
    print(f'[tiles] {len(reached & every)} of {len(every)} kernel instantiations reached')
    assert len(every) == 50
    assert every - reached == set(), sorted(every - reached)


def _k16_step(d, prods):
    """One k16 step under conv_oracle's model, for a non-negative accumulator d and products: the terms aligned to
    the largest exponent e and truncated to multiples of 2^(e - 25), summed exactly, the sum truncated to fp32."""
    terms = [d] + prods
    q = 2.0 ** (math.floor(math.log2(max(terms))) - 25)
    t = sum(math.floor(v / q) * q for v in terms)
    u = 2.0 ** (math.floor(math.log2(t)) - 23)
    return math.floor(t / u) * u


# (k16 steps, a): one product 1 and the others a 2^-24 per step, the latter just under, at, or half the fp32 ulp of
# the running sum.  The truncation they suffer is the largest the model allows per product.
@pytest.mark.parametrize('steps,a', [(8, 1.99), (8, 1.5), (32, 1.99), (8, 0.99)])
def test_k16_step_model(steps, a):
    """The device's k16 step is the one conv_oracle's bound assumes: after n steps the accumulator holds exactly what
    the model predicts, which is below the exact sum by up to a quarter fp32 ulp per product (more than the bound
    of a step that truncates only its exact sum allows), and the output is within the oracle's bound."""
    from shapy_b200 import ops
    cin = 16 * steps
    x = torch.full((1, 8, 8, cin), 2.0 ** -12)
    w = torch.full((16, cin, 1, 1), a * 2.0 ** -12)
    x[..., 0], w[:, 0] = 1.0, 1.0
    # the bias takes the 1 off, so the fp16 output holds D - 1 exactly (a multiple of 2^-24 below 2^-14)
    bias = torch.full((16,), -1.0)
    y = ops.conv_test(x.cuda(), w.cuda(), bias=bias.cuda(), relu=False, mode=0, engine=0)
    p = float(torch.tensor(a * 2.0 ** -12).half()) * 2.0 ** -12
    model = _k16_step(0.0, [1.0] + [p] * 15)
    for _ in range(steps - 1):
        model = _k16_step(model, [p] * 16)
    assert float(y[0, 0, 0, 0]) == model - 1.0, (float(y[0, 0, 0, 0]) / 2 ** -23, (model - 1) / 2 ** -23)
    ref = co.reference(x.cuda(), w.cuda(), bias=bias, mode=0)
    assert co.ratio(y, ref) <= 1.0, co.worst(y, ref)
