"""GPU: every network kernel alone against the float64 references of tests/kernel_refs.py, at the shapes where kernels
go wrong (channel and spatial tails, column windows inside wider tensors, partial batches, ring wrap-around), in every
launch schedule the product uses (SM limits of the overlapped predictor, PIFPAF_DW_CBF, PIFPAF_PDL,
PIFPAF_GEMM_RES_STAGES), the overlapped predictor against the sequential one, and a teacher-forced per-op check of
the real networks.

Single-op cases run one op in a net whose max_batch exceeds the batch.  Inputs are random bf16-exact values in every
column (the padding columns too: each weight there is zero, no op may rely on them being zero); every output tensor
and head buffer starts as kernel_refs.SENTINEL.  Inside its window an output must meet the float64 bound; everywhere
else -- other columns, images >= batch -- the sentinel must survive.  The worst err / bound of each op kind is printed
at the end of the module (run with -s)."""
import ctypes
import os

import numpy as np
import pytest
import torch

import kernel_refs as kr
import net_plan
from openpifpaf_b200 import _lib, constants, decoder, network, predictor
from oracle import net_oracle

pytestmark = pytest.mark.gpu

SLACK = {}          # op kind -> worst err / bound seen


def record(kind, ratio, what=''):
    SLACK[kind] = max(SLACK.get(kind, 0.0), ratio)
    assert ratio <= 1.0, f'{kind} {what}: err / bound = {ratio:.3g}'


@pytest.fixture(scope='module', autouse=True)
def slack_report():
    yield
    print('\nworst err / bound per op kind:')
    for k in sorted(SLACK):
        print(f'  {k:28s} {SLACK[k]:.3f}')


def ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def i32(v):
    return np.ascontiguousarray(v, dtype=np.int32)


def pad8(v):
    return (v + 7) // 8 * 8


def pad16(v):
    return (v + 15) // 16 * 16


def n_sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


class Case:
    """One net (max_batch images) with the given tensors; `inputs` are filled with random bf16 values, every other
    tensor with the sentinel.  emit(L, handle) adds the op(s)."""

    def __init__(self, max_batch, tensors, inputs, seed=0):
        self.mb, self.tensors = max_batch, list(tensors)
        self.rng = np.random.default_rng(seed)
        self.data = {}
        for t in range(len(self.tensors)):
            h, w, c = self.tensors[t]
            if t in inputs:
                self.data[t] = kr.random_bf16(self.rng, (max_batch, h, w, c))
            else:
                self.data[t] = np.full((max_batch, h, w, c), kr.SENTINEL, dtype=np.float32)

    def run(self, emit, batch, impl=0, sm_limit=0, images=None, u8=None):
        """-> (taps of every tensor over max_batch images, head buffers over max_batch images)"""
        L = _lib.lib()
        net = ctypes.c_void_p()
        _lib.check(L.pifpaf_net_create(ctypes.byref(net), 0, self.mb))
        try:
            tid = ctypes.c_int32()
            for t, (h, w, c) in enumerate(self.tensors):
                _lib.check(L.pifpaf_net_tensor(net, h, w, c, ctypes.byref(tid)))
                assert tid.value == t
                _lib.check(L.pifpaf_net_set_tensor(net, t, self.mb, ptr(self.data[t]), self.data[t].size))
            n_heads = emit(L, net) or 0
            heads = []
            for i in range(n_heads):
                p = ctypes.c_void_p()
                nf, nc, hh, ww = (ctypes.c_int32() for _ in range(4))
                _lib.check(L.pifpaf_net_head_output(net, i, ctypes.byref(p), ctypes.byref(nf), ctypes.byref(nc),
                                                    ctypes.byref(hh), ctypes.byref(ww)))
                v = torch.as_tensor(network._DevArray(p.value, (self.mb, nf.value, nc.value, hh.value, ww.value)),
                                    device='cuda:0')
                v.fill_(kr.SENTINEL)
                heads.append(v)
            if sm_limit:
                _lib.check(L.pifpaf_net_set_sm_limit(net, sm_limit))
            torch.cuda.synchronize()
            if u8 is not None:
                dev = torch.from_numpy(u8).cuda()
                m = (ctypes.c_float * 3)(*network.CompiledNet.IMAGE_MEAN)
                s = (ctypes.c_float * 3)(*network.CompiledNet.IMAGE_STD)
                _lib.check(L.pifpaf_net_forward_u8(net, dev.data_ptr(), batch, m, s, impl, None))
            else:
                dev = None if images is None else torch.from_numpy(images).cuda()
                _lib.check(L.pifpaf_net_forward(net, None if dev is None else dev.data_ptr(), batch, impl, None))
            torch.cuda.synchronize()
            taps = {}
            for t, (h, w, c) in enumerate(self.tensors):
                taps[t] = np.empty((self.mb, h, w, c), dtype=np.float32)
                _lib.check(L.pifpaf_net_tap_tensor(net, t, self.mb, ptr(taps[t]), taps[t].size))
            heads = [v.cpu().numpy() for v in heads]
        finally:
            L.pifpaf_net_destroy(net)
        return taps, heads


class Check:
    """Collects, per output tensor, the column windows an op owns and the comparisons inside them."""

    def __init__(self, kind, batch):
        self.kind, self.batch = kind, batch
        self.owned = {}           # tensor -> list of (c0, c1)
        self.cmp = []             # (tensor, c0, ref, bound, step)

    def own(self, t, c0, c1):
        self.owned.setdefault(t, []).append((c0, c1))

    def compare(self, t, c0, ref, bound, step=1):
        """columns c0, c0 + step, ... of tensor t hold ref (within bound)"""
        self.cmp.append((t, c0, ref, bound, step))

    def exact(self, t, c0, want, step=1):
        self.compare(t, c0, np.asarray(want, dtype=np.float64), np.zeros(np.shape(want)), step)

    def verify(self, taps, what=''):
        worst = 0.0
        for t, c0, ref, bound, step in self.cmp:
            n = ref.shape[-1]
            got = taps[t][:self.batch, ..., c0:c0 + step * (n - 1) + 1:step]
            worst = max(worst, kr.worst_ratio(got, ref, bound))
        for t, wins in self.owned.items():
            out = taps[t]
            mask = np.ones(out.shape[-1], dtype=bool)
            for c0, c1 in wins:
                mask[c0:c1] = False
            assert (out[self.batch:] == kr.SENTINEL).all(), f'{self.kind} {what}: wrote image >= batch of tensor {t}'
            stray = out[:self.batch][..., mask] != kr.SENTINEL
            assert not stray.any(), f'{self.kind} {what}: wrote {int(stray.sum())} values outside its columns of tensor {t}'
        record(self.kind, worst, what)
        return worst


# ---------------------------------------------------------------------------------------------------- depthwise
# (H, W, channels, kernel, stride, pad, in_off, out_off, relu, batch, max_batch)
DW5_CASES = [
    (1, 1, 8, 5, 1, 2, 0, 0, 1, 1, 2),
    (3, 5, 24, 5, 2, 2, 8, 16, 0, 2, 3),
    (8, 16, 72, 5, 1, 2, 0, 8, 1, 3, 4),          # exactly one 8 x 16 tile
    (16, 32, 176, 5, 2, 2, 0, 0, 0, 2, 3),        # exactly one stride-2 tile
    (16, 32, 176, 5, 1, 1, 16, 0, 1, 1, 2),
    (9, 17, 20, 5, 1, 0, 0, 0, 0, 4, 5),          # pad 0, channel tail inside one 8-channel vector
    (9, 17, 348, 5, 1, 2, 0, 0, 0, 2, 3),         # 6 channel blocks, the last one partial
    (9, 17, 348, 5, 2, 0, 0, 24, 1, 3, 5),
    (37, 23, 696, 5, 2, 2, 0, 0, 0, 2, 3),        # 11 channel blocks (cblks > 8)
    (37, 23, 696, 5, 1, 2, 8, 0, 1, 1, 2),
    (12, 9, 8, 5, 2, 1, 0, 0, 0, 4, 5),
    (161, 161, 176, 5, 1, 2, 0, 0, 0, 2, 3),      # many items per CTA: the slot ring wraps many times
    (161, 161, 348, 5, 2, 2, 0, 0, 1, 5, 6),
]
# the other depthwise kernels: 3x3 runs DW_TMA[DW_K3_*], k_dwconv takes 7x7, dilations other than 2 and every
# kernel but the 5x5 under gemm_impl = 1.  Optional trailing fields: (dilation, gemm_impl)
DWK_CASES = [
    (13, 11, 20, 3, 1, 1, 0, 0, 1, 2, 3),
    (13, 11, 36, 3, 2, 1, 8, 16, 0, 1, 2),
    (17, 19, 44, 7, 1, 3, 0, 0, 0, 2, 3),
    (17, 19, 12, 7, 2, 3, 0, 8, 1, 3, 4),
    (6, 5, 72, 3, 2, 0, 0, 0, 1, 1, 2),
    (13, 11, 24, 3, 1, 1, 8, 0, 2, 2, 3),              # ReLU6
    (21, 19, 20, 3, 1, 3, 0, 8, 1, 2, 3, 3, 0),         # dilation 3
    (23, 21, 36, 5, 1, 6, 0, 0, 0, 1, 2, 3, 0),         # 5x5, dilation 3
    (17, 15, 44, 5, 1, 8, 8, 0, 1, 2, 3, 4, 0),         # 5x5, dilation 4
    (12, 14, 24, 5, 2, 2, 0, 0, 2, 2, 3),               # 5x5 with ReLU6: k_dwconv5
    (13, 11, 20, 3, 1, 1, 0, 16, 1, 2, 3, 1, 1),        # 3x3 under gemm_impl = 1: k_dwconv, stride 1
    (13, 11, 36, 3, 2, 1, 8, 0, 2, 1, 2, 1, 1),         # ... stride 2
    (29, 27, 72, 7, 2, 3, 0, 0, 1, 2, 3, 1, 1),
]


def dw_case(H, W, C, k, stride, pad, in_off, out_off, relu, batch, mb, dil=1, impl=0, seed=0):
    Ho, Wo = kr.out_hw(H, W, (k - 1) * dil + 1, stride, pad)
    cin = pad16(in_off + pad8(C) + 8)
    cout = pad16(out_off + pad8(C) + 16)
    case = Case(mb, [(H, W, cin), (Ho, Wo, cout)], inputs={0}, seed=seed)
    rng = np.random.default_rng(seed + 1)
    w = (rng.standard_normal((C, k, k)) / k).astype(np.float32)        # f32 weights: not rounded to bf16
    b = rng.standard_normal(C).astype(np.float32)

    def emit(L, net):
        _lib.check(L.pifpaf_net_dwconv_dilated(net, 0, in_off, C, k, stride, pad, ptr(w), ptr(b), relu, 1, out_off,
                                               dil))

    x = case.data[0][:batch, ..., in_off:in_off + C]
    ref, mag = kr.conv_ref(x, w.reshape(C, 1, k, k), b, stride, pad, groups=C, dilation=dil)
    ref, mag = kr.epilogue(ref, mag, relu)
    chk = Check(dw_label(C, k, stride, relu, dil, impl), batch)
    chk.own(1, out_off, out_off + pad8(C))
    chk.compare(1, out_off, ref, kr.bf16_bound(ref, mag, k * k))
    if pad8(C) > C:       # padding channels: zero weight and bias
        chk.exact(1, out_off + C, np.zeros(ref.shape[:-1] + (pad8(C) - C,)))
    return case, emit, chk


def dw_label(C, k, stride, relu, dil=1, impl=0):
    """op kind of a depthwise case: its geometry and the kernel net.cu launches for it"""
    return 'dwconv k%d s%d%s %s' % (k, stride, ' d%d' % dil if dil > 1 else '',
                                    net_plan.dw_kernel(C, k, stride, relu, dil, gemm_impl=impl))


def dw_id(c):
    return 'H%dW%d-C%d-k%ds%dp%d-in%d-out%d-relu%d-B%dof%d' % c[:11] + ('-d%d-impl%d' % c[11:] if len(c) > 11 else '')


@pytest.mark.parametrize('impl', [0, 1], ids=['tma', 'simt'])
@pytest.mark.parametrize('c', DW5_CASES, ids=dw_id)
def test_dwconv5_matches_float64(c, impl):
    case, emit, chk = dw_case(*c, impl=impl)
    taps, _ = case.run(emit, c[9], impl=impl)
    print(dw_id(c), impl, '%.3f' % chk.verify(taps, dw_id(c)))


@pytest.mark.parametrize('c', DWK_CASES, ids=dw_id)
def test_dwconv_generic_matches_float64(c):
    case, emit, chk = dw_case(*c)
    taps, _ = case.run(emit, c[9], impl=c[12] if len(c) > 12 else 0)
    print(dw_id(c), '%.3f' % chk.verify(taps, dw_id(c)))


@pytest.mark.parametrize('C', [348, 696])
def test_dwconv5_stride2_channel_block_fastest(C, monkeypatch):
    """PIFPAF_DW_CBF=1: C = 348 takes the channel-block-fastest kernel (weights staged in shared memory), C = 696 does
    not fit and falls back.  Both meet the bound and equal the default order bit for bit (same per-lane FMA chain)."""
    c = (37, 41, C, 5, 2, 2, 0, 0, 1, 3, 4)
    case, emit, chk = dw_case(*c)
    monkeypatch.delenv('PIFPAF_DW_CBF', raising=False)
    base, _ = case.run(emit, 3)
    monkeypatch.setenv('PIFPAF_DW_CBF', '1')
    taps, _ = case.run(emit, 3)
    chk.kind += ' cbf'
    print('cbf C=%d %.3f' % (C, chk.verify(taps)))
    np.testing.assert_array_equal(taps[1], base[1])


# ---------------------------------------------------------------------------------------------------- fused dw -> 1x1
fused_rings = net_plan.fused_rings


# (H, W, channels, n_out, pieces [(count, dest, col)], dest widths, dw_relu, relu, batch, max_batch)
FUSED_CASES = [
    (9, 17, 72, 16, [(16, 0, 16)], [48], 0, 1, 1, 2),
    (8, 16, 176, 48, [(16, 0, 0), (32, 1, 16)], [32, 64], 1, 1, 2, 3),
    (13, 21, 176, 176, [(64, 0, 32), (48, 1, 0), (64, 2, 16)], [112, 64, 96], 0, 1, 2, 3),
    (20, 37, 348, 192, [(96, 0, 0), (96, 1, 16)], [112, 128], 0, 0, 1, 2),
    (11, 19, 72, 208, [(208, 0, 0)], [224], 0, 1, 3, 4),                        # two column blocks
    (9, 17, 348, 352, [(112, 0, 16), (128, 1, 0), (112, 2, 32)], [128, 144, 160], 0, 1, 2, 3),
    (33, 35, 176, 512, [(256, 0, 0), (256, 1, 0)], [272, 256], 1, 1, 2, 3),     # three column blocks of 176
    (9, 11, 696, 192, [(192, 0, 16)], [224], 0, 1, 2, 3),
    (9, 11, 1000, 192, [(96, 0, 0), (96, 1, 0)], [96, 112], 0, 1, 1, 2),
    (9, 11, 1024, 192, [(192, 0, 0)], [192], 0, 0, 2, 3),
    (161, 161, 176, 176, [(80, 0, 0), (96, 1, 16)], [96, 112], 0, 1, 2, 3),     # ~400 patches per image
]


def fused_id(c):
    return 'H%dW%d-C%d-N%d-%dpieces-rings%d%d-B%dof%d' % (c[:4] + (len(c[4]),) + fused_rings(c[2], c[3]) + c[8:])


def test_fused_cases_reach_every_ring_depth():
    assert {fused_rings(c[2], c[3]) for c in FUSED_CASES} == {(3, 2), (2, 2), (2, 1), (1, 1)}


def fused_case(H, W, C, N, pieces, widths, dw_relu, relu, batch, mb, seed=0):
    cin = pad16(pad8(C) + 8)
    tensors = [(H, W, cin)] + [(H, W, wd) for wd in widths]
    case = Case(mb, tensors, inputs={0}, seed=seed)
    rng = np.random.default_rng(seed + 2)
    dw_w = (rng.standard_normal((C, 5, 5)) / 5).astype(np.float32)
    dw_b = rng.standard_normal(C).astype(np.float32)
    w = kr.random_bf16(rng, (N, C), 1 / np.sqrt(C))
    b = rng.standard_normal(N).astype(np.float32)
    col0 = np.cumsum([0] + [p[0] for p in pieces])[:-1]
    pc = [i32(col0), i32([p[0] for p in pieces]), i32([p[1] + 1 for p in pieces]), i32([p[2] for p in pieces])]

    def emit(L, net):
        _lib.check(L.pifpaf_net_dw_conv1x1_scatter(net, 0, 0, C, 5, 1, 2, ptr(dw_w), ptr(dw_b), dw_relu, N, ptr(w),
                                                   ptr(b), relu, len(pieces), *[ptr(a) for a in pc]))

    ref, bound = kr.dw_gemm_ref(case.data[0][:batch, ..., :C], dw_w, dw_b, dw_relu, w, b, relu)
    chk = Check('dw_gemm', batch)
    for c0, (cnt, d, col) in zip(col0, pieces):
        chk.own(d + 1, col, col + cnt)
        chk.compare(d + 1, col, ref[..., c0:c0 + cnt], bound[..., c0:c0 + cnt])
    return case, emit, chk


@pytest.mark.parametrize('c', FUSED_CASES, ids=fused_id)
def test_fused_dw_gemm_matches_float64(c):
    case, emit, chk = fused_case(*c)
    taps, _ = case.run(emit, c[8])
    print(fused_id(c), '%.3f' % chk.verify(taps, fused_id(c)))


# ---------------------------------------------------------------------------------------------------- dense conv
# (H, W, c_in, kernel, stride, pad, n_out, in_off, residual col (None: no residual), relu, out_off, batch, max_batch)
# n_out whose tiles are 16, 32, ..., 256 columns wide: every (column groups, last group width) instantiation of
# k_gemm_wg, in order (1 x 16 ... 4 x 64); N = bn - 10 leaves a partial last 16-column group
TILE_WIDTHS = [16, 22, 44, 64, 70, 92, 108, 124, 140, 150, 174, 188, 208, 214, 236, 256]

CONV_CASES = [
    (9, 11, 64, 1, 2, 0, 32, 0, None, 0, 0, 1, 2),        # 1x1 stride 2 (ResNet downsample)
    (17, 19, 64, 3, 1, 1, 64, 0, 16, 1, 0, 2, 3),         # residual at a column offset
    (17, 19, 72, 3, 2, 1, 80, 8, None, 1, 16, 2, 3),      # K tail, column windows
    (6, 7, 3, 3, 1, 0, 16, 0, None, 0, 0, 1, 2),          # c_in 3; Ho x Wo smaller than one 8 x 16 patch
    (13, 15, 200, 5, 1, 2, 48, 0, 8, 1, 0, 2, 2),
    (23, 29, 64, 7, 2, 3, 272, 0, None, 1, 0, 1, 2),
    (21, 37, 72, 5, 2, 0, 112, 0, 0, 0, 0, 2, 3),         # residual, no ReLU
    (9, 9, 200, 3, 2, 2, 24, 0, None, 0, 32, 3, 4),
    (10, 12, 64, 3, 1, 3, 16, 0, None, 1, 0, 1, 2),       # pad 3 > k / 2
    (57, 61, 64, 3, 1, 1, 128, 0, 0, 1, 0, 2, 3),         # 40 patches per image
    (11, 13, 136, 1, 1, 0, 120, 8, 24, 1, 0, 2, 3),       # 1x1 stride 1 with residual: the pointwise GEMM route
    (11, 13, 136, 1, 1, 0, 120, 8, 24, 0, 16, 2, 3),
    (15, 17, 128, 1, 2, 0, 96, 0, None, 1, 0, 2, 3),      # 2 K blocks: a 4-deep ring
    (17, 19, 64, 1, 2, 0, 128, 0, None, 1, 0, 2, 3),      # 1 K block: a 2-deep ring (ResNet's 128-wide downsample)
    # the pointwise plans of the shipped MobileNetV2 and ResNet-50 (tests/test_net_plan.py lists them)
    (9, 11, 160, 1, 1, 0, 960, 0, None, 2, 0, 2, 3),      # ReLU6, 4 x 240, resident 6
    (7, 9, 320, 1, 1, 0, 1280, 0, None, 2, 0, 2, 3),      # ReLU6, 5 x 256, streaming 4
    (9, 11, 576, 1, 1, 0, 96, 0, 0, 0, 0, 2, 3),          # residual, 96, resident 5
    (9, 11, 960, 1, 1, 0, 160, 0, 0, 0, 0, 2, 3),         # residual, 160, streaming 5
    (7, 9, 512, 1, 1, 0, 2048, 0, 0, 1, 0, 2, 3),         # residual, 8 x 256, streaming 4
    (9, 11, 256, 1, 1, 0, 1024, 0, 0, 1, 0, 2, 3),        # residual, 4 x 256, resident 4
    (9, 11, 64, 1, 1, 0, 256, 0, 0, 1, 0, 2, 3),          # residual, 256, resident 8
] + [
    # every instantiation of the pointwise route with the per-lane residual epilogue (activation codes 0 / 1 / 2)
    (11, 13, 136, 1, 1, 0, n, 8, 16, i % 3, 0, 2, 3) for i, n in enumerate(TILE_WIDTHS)
] + [
    # every instantiation of the implicit GEMM, 3x3 at stride 1 and 2: plain, ReLU6, residual (codes 0 / 1 / 2)
    (11, 13, 72, 3, 1 + i % 2, 1, n, 8, None, 1, 16, 2, 3) for i, n in enumerate(TILE_WIDTHS)
] + [
    (12, 10, 64, 3, 2 - i % 2, 1, n, 0, None, 2, 0, 1, 2) for i, n in enumerate(TILE_WIDTHS)
] + [
    (10, 13, 64, 3, 1 + i % 2, 1, n, 0, 8, i % 3, 0, 2, 3) for i, n in enumerate(TILE_WIDTHS)
]


def conv_id(c):
    return 'H%dW%d-cin%d-k%ds%dp%d-N%d-in%d-res%s-relu%d-out%d-B%dof%d' % c


def conv_case(H, W, c_in, k, stride, pad, N, in_off, res_col, relu, out_off, batch, mb, seed=0):
    Ho, Wo = kr.out_hw(H, W, k, stride, pad)
    tensors = [(H, W, pad16(in_off + c_in + 8)), (Ho, Wo, pad16(out_off + pad8(N) + 16))]
    inputs = {0}
    if res_col is not None:
        tensors.append((Ho, Wo, pad16(res_col + N + 8)))
        inputs.add(2)
    case = Case(mb, tensors, inputs=inputs, seed=seed)
    rng = np.random.default_rng(seed + 3)
    w = kr.random_bf16(rng, (N, c_in, k, k), (4 if relu == 2 else 1) / np.sqrt(c_in * k * k))     # ReLU6: past 6
    b = rng.standard_normal(N).astype(np.float32)

    def emit(L, net):
        _lib.check(L.pifpaf_net_conv(net, 0, in_off, c_in, k, stride, pad, N, ptr(w), ptr(b), relu, 1, out_off,
                                     -1 if res_col is None else 2, 0 if res_col is None else res_col))

    ref, mag = kr.conv_ref(case.data[0][:batch, ..., in_off:in_off + c_in], w, b, stride, pad)
    res = None if res_col is None else case.data[2][:batch, ..., res_col:res_col + N]
    ref, mag = kr.epilogue(ref, mag, relu, res)
    chk = Check('conv k%d' % k + (' relu6' if relu == 2 else ''), batch)
    chk.own(1, out_off, out_off + pad8(N))
    chk.compare(1, out_off, ref, kr.bf16_bound(ref, mag, c_in * k * k))
    if res_col is None and pad8(N) > N:
        chk.exact(1, out_off + N, np.zeros(ref.shape[:-1] + (pad8(N) - N,)))
    return case, emit, chk


@pytest.mark.parametrize('impl', [0, 1], ids=['wgmma', 'simt'])
@pytest.mark.parametrize('c', CONV_CASES, ids=conv_id)
def test_conv_matches_float64(c, impl):
    case, emit, chk = conv_case(*c)
    taps, _ = case.run(emit, c[11], impl=impl)
    print(conv_id(c), impl, '%.3f' % chk.verify(taps, conv_id(c)))


# ---------------------------------------------------------------------------------------------------- input conv
# (H, W, kernel, stride, pad, c_out, u8, batch, max_batch)
STEM_CASES = [
    (17, 19, 1, 1, 0, 8, False, 1, 2),
    (17, 19, 1, 1, 0, 8, True, 1, 2),
    (33, 31, 3, 2, 1, 24, False, 2, 3),
    (33, 31, 3, 2, 1, 24, True, 2, 3),
    (21, 25, 5, 1, 2, 64, False, 1, 2),
    (21, 25, 5, 2, 0, 64, True, 2, 2),
    (45, 47, 7, 2, 3, 64, False, 2, 2),
    (45, 47, 7, 2, 3, 80, False, 2, 3),       # 51 KB of weights in shared memory: past the default 48 KB
    (45, 47, 7, 2, 3, 80, True, 2, 3),
    (16, 16, 7, 1, 3, 20, True, 3, 4),
]


def stem_id(c):
    return 'H%dW%d-k%ds%dp%d-C%d-%s-B%dof%d' % (c[:6] + ('u8' if c[6] else 'f32',) + c[7:])


def stem_case(H, W, k, stride, pad, C, u8, batch, mb, seed=0):
    Ho, Wo = kr.out_hw(H, W, k, stride, pad)
    case = Case(mb, [(Ho, Wo, pad16(pad8(C) + 8))], inputs=set(), seed=seed)
    rng = np.random.default_rng(seed + 4)
    w = (rng.standard_normal((C, 3, k, k)) / k).astype(np.float32)
    b = rng.standard_normal(C).astype(np.float32)
    if u8:
        raw = rng.integers(0, 256, (batch, H, W, 3), dtype=np.uint8)
        x = kr.normalise_u8(raw, network.CompiledNet.IMAGE_MEAN, network.CompiledNet.IMAGE_STD)
        kw = {'u8': raw}
    else:
        images = rng.standard_normal((batch, 3, H, W)).astype(np.float32)
        x = images.transpose(0, 2, 3, 1)
        kw = {'images': images}

    def emit(L, net):
        _lib.check(L.pifpaf_net_input_conv(net, H, W, k, stride, pad, C, ptr(w), ptr(b), 1, 0))

    ref, mag = kr.conv_ref(x, w, b, stride, pad)
    ref, mag = kr.epilogue(ref, mag, True)
    chk = Check('input_conv', batch)
    chk.own(0, 0, pad8(C))
    chk.compare(0, 0, ref, kr.bf16_bound(ref, mag, 3 * k * k))
    if pad8(C) > C:
        chk.exact(0, C, np.zeros(ref.shape[:-1] + (pad8(C) - C,)))
    return case, emit, chk, kw


@pytest.mark.parametrize('c', STEM_CASES, ids=stem_id)
def test_input_conv_matches_float64(c):
    case, emit, chk, kw = stem_case(*c)
    taps, _ = case.run(emit, c[7], **kw)
    chk.kind += ' u8' if c[6] else ' f32'
    print(stem_id(c), '%.3f' % chk.verify(taps, stem_id(c)))


def test_input_conv_rejects_weights_past_shared_memory():
    """a 7x7 stem with 400 channels needs 235 KB of weights in shared memory: refused when the op is added"""
    L = _lib.lib()
    net = ctypes.c_void_p()
    _lib.check(L.pifpaf_net_create(ctypes.byref(net), 0, 1))
    try:
        tid = ctypes.c_int32()
        _lib.check(L.pifpaf_net_tensor(net, 8, 8, 400, ctypes.byref(tid)))
        w = np.zeros((400, 3, 7, 7), dtype=np.float32)
        b = np.zeros(400, dtype=np.float32)
        assert L.pifpaf_net_input_conv(net, 16, 16, 7, 2, 3, 400, ptr(w), ptr(b), 1, tid.value) == _lib.E_BADARG
        assert b'shared memory' in L.pifpaf_last_error()
        assert L.pifpaf_net_num_ops(net) == 0
    finally:
        L.pifpaf_net_destroy(net)


# ---------------------------------------------------------------------------------------------------- 1x1 GEMM
# (h, w, K, N, in_off, out_off, shuffle, relu, batch, max_batch)
GEMM_CASES = [
    (9, 11, 72, 96, 0, 16, False, 0, 2, 3),
    (12, 12, 174, 174, 176, 0, False, 0, 1, 3),
    (13, 9, 256, 256, 0, 0, False, 1, 2, 4),
    (9, 11, 352, 348, 0, 0, True, 0, 2, 3),
    (41, 41, 1392, 240, 0, 32, False, 0, 1, 2),        # streaming weights
    (64, 64, 352, 176, 0, 0, False, 0, 3, 4),
    (161, 161, 176, 174, 0, 0, True, 1, 1, 2),         # pass-through double buffer wraps
    # streaming weights (K = 1392) at ring depths 8 / 7 / 6, and 2 (a 224-column shuffle tile and its pass-through buffer)
    (17, 19, 1392, 64, 0, 0, False, 0, 1, 2),
    (17, 19, 1392, 96, 0, 16, False, 1, 2, 3),
    (17, 19, 1392, 128, 0, 0, False, 0, 1, 2),
    (17, 19, 1392, 224, 0, 0, True, 1, 1, 2),
    # shuffle with the pass-through tile read per lane: 240 / 256-column tiles, and 4 blocks of 224 columns whose bias
    # and scatter tables leave no room for the double buffer
    (13, 11, 176, 236, 0, 0, True, 0, 2, 3),
    (13, 11, 176, 256, 0, 0, True, 1, 2, 3),
    (9, 11, 96, 896, 0, 0, True, 1, 2, 3),
    # the shuffle plans of the shipped k16 / k30 stage GEMMs without src_tma (tests/test_net_plan.py lists them)
    (9, 11, 704, 696, 0, 0, True, 1, 2, 3),            # 240 x 3, streaming 4
    (9, 11, 512, 512, 0, 0, True, 1, 2, 3),            # 256 x 2, streaming 4
    (9, 11, 256, 256, 0, 0, True, 0, 2, 3),            # 256, resident 4
] + [
    (9, 11, 72, n, 0, 0, True, i % 2, 2, 3) for i, n in enumerate(TILE_WIDTHS[:14])     # shuffle, src_tma
] + [
    (9, 11, 72, n, 0, 16 * (i % 2), False, 2, 2, 3) for i, n in enumerate(TILE_WIDTHS)  # ReLU6: per-lane epilogue
]


def gemm_id(c):
    return 'hw%dx%d-K%d-N%d-in%d-out%d-%s-relu%d-B%dof%d' % (c[:6] + ('shuffle' if c[6] else 'plain',) + c[7:])


def gemm_case(h, w, K, N, in_off, out_off, shuffle, relu, batch, mb, seed=0):
    tensors = [(h, w, pad16(in_off + K + 8)), (h, w, pad16(2 * N if shuffle else out_off + pad8(N)) + 16)]
    inputs = {0}
    if shuffle:
        tensors.append((h, w, pad16(N)))
        inputs.add(2)
    case = Case(mb, tensors, inputs=inputs, seed=seed)
    rng = np.random.default_rng(seed + 5)
    wt = kr.random_bf16(rng, (N, K), (4 if relu == 2 else 1) / np.sqrt(K))      # ReLU6: outputs past 6
    b = rng.standard_normal(N).astype(np.float32)

    def emit(L, net):
        _lib.check(L.pifpaf_net_conv1x1(net, 0, in_off, K, N, ptr(wt), ptr(b), relu, 1, out_off,
                                        2 if shuffle else -1, 0))

    ref, mag = kr.conv_ref(case.data[0][:batch, ..., in_off:in_off + K], wt[:, :, None, None], b, 1, 0)
    ref, mag = kr.epilogue(ref, mag, relu)
    bound = kr.bf16_bound(ref, mag, K)
    chk = Check('gemm ' + ('shuffle' if shuffle else 'plain') + (' relu6' if relu == 2 else ''), batch)
    if shuffle:
        chk.own(1, 0, 2 * N)
        chk.compare(1, 1, ref, bound, step=2)
        chk.exact(1, 0, case.data[2][:batch, ..., :N], step=2)
    else:
        chk.own(1, out_off, out_off + pad8(N))
        chk.compare(1, out_off, ref, bound)
        if pad8(N) > N:
            chk.exact(1, out_off + N, np.zeros(ref.shape[:-1] + (pad8(N) - N,)))
    return case, emit, chk


@pytest.mark.parametrize('impl', [0, 1], ids=['wgmma', 'simt'])
@pytest.mark.parametrize('c', GEMM_CASES, ids=gemm_id)
def test_conv1x1_matches_float64_outside_untouched(c, impl):
    case, emit, chk = gemm_case(*c)
    taps, _ = case.run(emit, c[8], impl=impl)
    print(gemm_id(c), impl, '%.3f' % chk.verify(taps, gemm_id(c)))


# (h, w, K, n_out, pieces [(count, dest, col)], dest widths, relu, batch, max_batch); resident / streaming weight tile
SCATTER_CASES = [
    (9, 11, 72, 48, [(16, 0, 16), (16, 1, 0), (16, 2, 32)], [48, 32, 64], 0, 2, 3),
    (17, 13, 176, 368, [(112, 0, 0), (128, 1, 16), (128, 2, 0)], [128, 160, 144], 0, 1, 2),    # 2 x 192, resident
    (17, 13, 1392, 368, [(176, 0, 32), (192, 1, 0)], [224, 208], 1, 2, 3),                     # streaming
    (41, 43, 352, 176, [(96, 0, 0), (80, 1, 16)], [112, 112], 1, 2, 3),
    (41, 43, 416, 176, [(176, 0, 16)], [192], 0, 1, 2),
    (33, 35, 352, 192, [(192, 0, 0)], [208], 1, 3, 4),
]


def scatter_id(c):
    return 'hw%dx%d-K%d-N%d-%dpieces-relu%d-B%dof%d' % (c[:4] + (len(c[4]),) + c[6:])


def scatter_case(h, w, K, N, pieces, widths, relu, batch, mb, seed=0):
    tensors = [(h, w, pad16(K + 8))] + [(h, w, wd) for wd in widths]
    case = Case(mb, tensors, inputs={0}, seed=seed)
    rng = np.random.default_rng(seed + 6)
    wt = kr.random_bf16(rng, (N, K), 1 / np.sqrt(K))
    b = rng.standard_normal(N).astype(np.float32)
    col0 = np.cumsum([0] + [p[0] for p in pieces])[:-1]
    pc = [i32(col0), i32([p[0] for p in pieces]), i32([p[1] + 1 for p in pieces]), i32([p[2] for p in pieces])]

    def emit(L, net):
        _lib.check(L.pifpaf_net_conv1x1_scatter(net, 0, 0, K, N, ptr(wt), ptr(b), relu, len(pieces),
                                                *[ptr(a) for a in pc]))

    ref, mag = kr.conv_ref(case.data[0][:batch, ..., :K], wt[:, :, None, None], b, 1, 0)
    ref, mag = kr.epilogue(ref, mag, relu)
    bound = kr.bf16_bound(ref, mag, K)
    chk = Check('gemm scatter', batch)
    for c0, (cnt, d, col) in zip(col0, pieces):
        chk.own(d + 1, col, col + cnt)
        chk.compare(d + 1, col, ref[..., c0:c0 + cnt], bound[..., c0:c0 + cnt])
    return case, emit, chk


@pytest.mark.parametrize('impl', [0, 1], ids=['wgmma', 'simt'])
@pytest.mark.parametrize('c', SCATTER_CASES, ids=scatter_id)
def test_conv1x1_scatter_matches_float64(c, impl):
    case, emit, chk = scatter_case(*c)
    taps, _ = case.run(emit, c[7], impl=impl)
    print(scatter_id(c), impl, '%.3f' % chk.verify(taps, scatter_id(c)))


@pytest.mark.parametrize('c', SCATTER_CASES[3:5], ids=scatter_id)
def test_gemm_res_stages_retiling(c, monkeypatch):
    """PIFPAF_GEMM_RES_STAGES=5 splits a weights-resident tile into narrower column blocks: same bound, and the same
    bits (every output column still sums its K blocks in the same order)"""
    case, emit, chk = scatter_case(*c)
    monkeypatch.delenv('PIFPAF_GEMM_RES_STAGES', raising=False)
    base, _ = case.run(emit, c[7])
    monkeypatch.setenv('PIFPAF_GEMM_RES_STAGES', '5')
    taps, _ = case.run(emit, c[7])
    chk.kind += ' res_stages=5'
    print(scatter_id(c), 'res_stages=5 %.3f' % chk.verify(taps, scatter_id(c)))
    for t in base:
        np.testing.assert_array_equal(taps[t], base[t])


# ---------------------------------------------------------------------------------------------------- heads
WHOLEBODY = ((133, 1, 1, 1), (160, 1, 2, 2))       # 133 x 5 + 160 x 8 = 1945 columns
# (h, w, K, heads [(n_fields, n_conf, n_vec, n_scales)] or 'all' (one head with every comp op), batch, max_batch,
# optional upsample stride); a head has 1 + n_conf + 2 n_vec + n_scales components, each of up^2 conv columns
HEADS_CASES = [
    (9, 13, 136, ((17, 1, 1, 1), (19, 1, 2, 2)), 2, 3),     # N = 237; 117 pixels per image: tiles span two images
    (9, 11, 200, WHOLEBODY, 2, 3),
    (5, 7, 72, 'all', 3, 4),
    (16, 8, 64, ((3, 1, 1, 1),), 1, 2),                      # N = 15, exactly one 128-row tile per image
    (7, 9, 256, ((3, 1, 1, 1),), 2, 3),                      # K = 256: an 8-deep ring
    (7, 9, 256, ((19, 1, 1, 1),), 2, 3),                     # 96-column tile: 7 deep
    (7, 9, 256, ((25, 1, 1, 1),), 2, 3),                     # 128: 6 deep
    (7, 9, 256, ((35, 1, 1, 1),), 2, 3),                     # 176: 5 deep
    # several n blocks, a 5-component field straddling each block boundary (up = 1, 2), and a 3 x 3 sub-pixel group
    # straddling it (up = 3: 45 columns per field, 160-column blocks)
    (6, 7, 72, ((37, 1, 1, 1),), 2, 3, 2),
    (5, 6, 72, ((7, 1, 1, 1),), 2, 3, 3),
    (5, 6, 136, ((17, 1, 1, 1), (19, 1, 2, 2)), 1, 2, 3),
] + [
    (7, 5, 72, (((bn - 3) // 5, 1, 1, 1),), 2, 3) for bn in range(16, 257, 16)     # every instantiation
] + [
    (5, 4, 72, ((bn // 8, 1, 0, 0),), 2, 3, 2) for bn in range(16, 257, 16)        # upsampled, every instantiation
]


def heads_id(c):
    return 'hw%dx%d-K%d-%s-B%dof%d' % (c[0], c[1], c[2], 'all' if c[3] == 'all' else 'x'.join(str(h[0]) for h in c[3]),
                                       c[4], c[5]) + ('-up%d' % c[6] if len(c) > 6 else '')


def heads_case(h, w, K, spec, batch, mb, up=1, seed=0):
    if spec == 'all':
        n_fields, n_comp, ops = [3], [6], [0, 1, 2, 3, 4, 1]
    else:
        n_fields = [s[0] for s in spec]
        ops_h = [network.head_ops(s[1], s[2], s[3], (True,) * s[2]) for s in spec]
        n_comp = [len(o) for o in ops_h]
        ops = [o for oh in ops_h for o in oh]
    N = sum(f * c for f, c in zip(n_fields, n_comp)) * up * up
    case = Case(mb, [(h, w, pad16(K + 8))], inputs={0}, seed=seed)
    rng = np.random.default_rng(seed + 7)
    wt = kr.random_bf16(rng, (N, K), 2 / np.sqrt(K))
    b = rng.standard_normal(N).astype(np.float32)

    def emit(L, net):
        n = len(n_fields)
        _lib.check(L.pifpaf_net_heads_upsampled(net, 0, K, n, i32(n_fields).ctypes.data_as(ctypes.c_void_p),
                                                i32(n_comp).ctypes.data_as(ctypes.c_void_p),
                                                i32(ops).ctypes.data_as(ctypes.c_void_p), up, ptr(wt), ptr(b)))
        return n

    refs = kr.heads_ref(case.data[0][:batch, ..., :K], wt, b, n_fields, n_comp, ops, up)
    return case, emit, refs


def verify_heads(heads, refs, batch, what='', kind='heads'):
    worst = 0.0
    for hb, (ref, bound) in zip(heads, refs):
        assert (hb[batch:] == kr.SENTINEL).all(), f'heads {what}: wrote image >= batch'
        worst = max(worst, kr.worst_ratio(hb[:batch], ref, bound))
    record(kind, worst, what)
    return worst


@pytest.mark.parametrize('impl', [0, 1], ids=['wgmma', 'simt'])
@pytest.mark.parametrize('c', HEADS_CASES, ids=heads_id)
def test_heads_match_float64(c, impl):
    case, emit, refs = heads_case(*c)
    _, heads = case.run(emit, c[4], impl=impl)
    kind = 'heads upsampled' if len(c) > 6 else 'heads'
    print(heads_id(c), impl, '%.3f' % verify_heads(heads, refs, c[4], heads_id(c), kind))


# ---------------------------------------------------------------------------------------------------- schedules
SCHEDULE_CASES = {           # name -> (case factory, gemm_impl)
    'dwconv5 s1': (lambda: dw_case(161, 161, 176, 5, 1, 2, 0, 0, 0, 2, 3), 0),
    'dwconv5 s2': (lambda: dw_case(161, 161, 348, 5, 2, 2, 0, 0, 1, 2, 3), 0),
    'dw_gemm 1 block': (lambda: fused_case(*FUSED_CASES[-1]), 0),
    'dw_gemm 3 blocks': (lambda: fused_case(*FUSED_CASES[6]), 0),
    'conv 3x3': (lambda: conv_case(*CONV_CASES[9]), 0),
    'gemm shuffle': (lambda: gemm_case(*GEMM_CASES[6]), 0),
    'gemm plain': (lambda: gemm_case(*GEMM_CASES[5]), 0),
    'gemm scatter resident': (lambda: scatter_case(*SCATTER_CASES[5]), 0),
    'gemm scatter streaming': (lambda: scatter_case(*SCATTER_CASES[2]), 0),
    'heads': (lambda: heads_case(41, 41, 136, ((17, 1, 1, 1), (19, 1, 2, 2)), 3, 3), 0),
    'heads upsampled': (lambda: heads_case(21, 23, 72, ((7, 1, 1, 1),), 3, 3, 3), 0),
    'conv 3x3 4 groups residual relu6': (lambda: conv_case(41, 43, 64, 3, 2, 1, 236, 0, 8, 2, 0, 2, 3), 0),
    'conv 1x1 residual': (lambda: conv_case(57, 61, 136, 1, 1, 0, 188, 8, 16, 1, 0, 2, 3), 0),
    'gemm relu6': (lambda: gemm_case(64, 64, 352, 214, 0, 16, False, 2, 3, 4), 0),
    'gemm shuffle lane src': (lambda: gemm_case(61, 67, 176, 256, 0, 0, True, 1, 2, 3), 0),
    'gemm streaming 8 stages': (lambda: gemm_case(41, 41, 1392, 64, 0, 0, False, 0, 2, 3), 0),
    'input_conv': (lambda: stem_case(161, 161, 3, 2, 1, 24, False, 3, 3), 0),
    # grid-stride kernels whose grids also follow the SM count: k_dwconv5, k_dwconv, k_gemm_simt
    'dwconv5 s1 simt': (lambda: dw_case(61, 67, 176, 5, 1, 2, 0, 0, 0, 2, 3, impl=1), 1),
    'dwconv5 s2 simt': (lambda: dw_case(61, 67, 348, 5, 2, 2, 0, 0, 1, 2, 3, impl=1), 1),
    'dwconv k3 s2 tma': (lambda: dw_case(61, 67, 72, 3, 2, 1, 0, 0, 1, 2, 3), 0),
    'dwconv k7 generic': (lambda: dw_case(61, 67, 72, 7, 2, 3, 0, 0, 1, 2, 3), 0),
    'dwconv k3 d3 generic': (lambda: dw_case(61, 67, 40, 3, 1, 3, 0, 0, 1, 2, 3, 3), 0),
    'conv 3x3 simt': (lambda: conv_case(*CONV_CASES[9]), 1),
    'gemm plain simt': (lambda: gemm_case(*GEMM_CASES[5]), 1),
    'gemm scatter simt': (lambda: scatter_case(*SCATTER_CASES[1]), 1),
    'heads simt': (lambda: heads_case(41, 41, 136, ((17, 1, 1, 1), (19, 1, 2, 2)), 3, 3), 1),
}


@pytest.mark.parametrize('name', list(SCHEDULE_CASES))
def test_sm_limit_is_bitwise_invariant(name):
    """grids capped at 1, 2, 7, n_sm - 4 and n_sm - 8 SMs (the overlapped predictor's limits): every persistent CTA
    walks more tiles and every ring wraps differently, every grid-stride thread takes more items; the outputs stay
    identical bit for bit"""
    factory, impl = SCHEDULE_CASES[name]
    made = factory()
    case, emit = made[0], made[1]
    kw = made[3] if len(made) == 4 else {}
    batch = case.mb if name.startswith(('heads', 'input_conv')) else case.mb - 1
    base_t, base_h = case.run(emit, batch, impl=impl, **kw)
    for lim in (1, 2, 7, n_sm() - 4, n_sm() - 8):
        taps, heads = case.run(emit, batch, impl=impl, sm_limit=lim, **kw)
        for t in base_t:
            assert np.array_equal(taps[t], base_t[t]), (name, lim, t)
        for a, b in zip(heads, base_h):
            assert np.array_equal(a, b), (name, lim)


def test_pdl_off_is_bitwise_invariant(monkeypatch):
    """PIFPAF_PDL=0 (plain stream order between the ops) gives the fields of the PDL schedule bit for bit"""
    plan = network.random_plan('shufflenetv2k16', seed=3)
    x = torch.randn(3, 3, 129, 161, generator=torch.Generator().manual_seed(4)).cuda()
    monkeypatch.delenv('PIFPAF_PDL', raising=False)
    net = network.CompiledNet(plan, 129, 161, 4)
    want = [t.clone() for t in net.forward(x)]
    net.close()
    monkeypatch.setenv('PIFPAF_PDL', '0')
    net = network.CompiledNet(plan, 129, 161, 4)
    got = [t.clone() for t in net.forward(x)]
    net.close()
    for a, b in zip(got, want):
        assert torch.isfinite(a).all() and torch.equal(a, b)


# ---------------------------------------------------------------------------------------------------- overlapped predictor
@pytest.fixture(scope='module')
def k16_plan():
    """k16 whose heads emit image-dependent poses: the head weights are scaled down so that the confidences sit around
    sigmoid(-2) and the image moves them a little (a random-init net at full scale finds no poses)"""
    plan = network.random_plan('shufflenetv2k16', seed=0, confidence_bias=-2.0)
    for hd in plan['heads']:
        hd['w'] = hd['w'] * np.float32(0.06)
    return plan


@pytest.mark.parametrize('reserve', [None, 4, 8], ids=['policy', 'reserve4', 'reserve8'])
@pytest.mark.parametrize('max_batch', [16, 32])
def test_overlapped_predictor_equals_sequential(k16_plan, max_batch, reserve, monkeypatch):
    """Predictor(overlap_decode=True) -- double-buffered head outputs, the decode of step i on its own stream under
    the forward of step i + 1, the forward's grids capped below the SM count -- yields, step by step, the annotations
    and fields of the sequential predictor, bit for bit.  A decode that read a head-output set a later forward had
    already overwritten would change the annotations: every step has some, and they differ from step to step."""
    # the random-init poses score below the default instance threshold (0.15); keep them all
    monkeypatch.setattr(decoder.NMSKeypoints, '_instance_threshold', 0.0)
    H = W = 129
    g = torch.Generator().manual_seed(max_batch)
    hosts = [torch.randn(max_batch, 3, H, W, generator=g).pin_memory() for _ in range(5)]
    seq_net = network.CompiledNet(k16_plan, H, W, max_batch)
    seq = predictor.Predictor(seq_net, constants.COCO_N_KEYPOINTS, constants.COCO_PERSON_SKELETON)
    want, want_fields = [], []
    for hst in hosts:
        want.append(seq.batch(hst))
        torch.cuda.synchronize()
        want_fields.append([t.clone() for t in seq_net.forward(hst.cuda())])
        torch.cuda.synchronize()        # the predictor's own stream does not wait for the default stream
    seq.close()
    ovl_net = network.CompiledNet(k16_plan, H, W, max_batch)
    ovl = predictor.Predictor(ovl_net, constants.COCO_N_KEYPOINTS, constants.COCO_PERSON_SKELETON,
                              overlap_decode=True, reserve_sms=reserve)
    dev = [h.cuda() for h in hosts]
    torch.cuda.synchronize()
    got, got_fields = [], []
    outstanding = 0
    with torch.cuda.stream(ovl.stream):
        for d in dev:
            ovl.batch_device(d)
            got_fields.append([t.clone() for t in ovl_net._head_views(max_batch)])
            ovl.decoder.fetch_begin(stream=ovl.result_stream())
            outstanding += 1
            if outstanding == 2:            # step i is fetched after step i + 1 has been enqueued
                got.append(ovl.decoder.fetch_end())
                outstanding -= 1
        got.append(ovl.decoder.fetch_end())
        ovl.join()
    torch.cuda.synchronize()
    last = [t.clone() for t in ovl_net._head_views(max_batch)]
    ovl.close()
    assert len(got) == len(want) == 5
    n_ann = []
    for step, (rw, rg) in enumerate(zip(want, got)):
        assert len(rw) == len(rg) == max_batch
        for (aw, iw), (ag, ig) in zip(rw, rg):
            assert torch.equal(aw, ag) and torch.equal(iw, ig), step
        n_ann.append(sum(int(aw.shape[0]) for aw, _ in rw))
        for a, b in zip(got_fields[step], want_fields[step]):
            assert torch.equal(a, b), step
    for a, b in zip(last, want_fields[-1]):
        assert torch.equal(a, b)
    print('overlap', max_batch, reserve, 'annotations per step', n_ann)
    assert min(n_ann) > 0
    for step in range(1, len(want)):      # the poses follow the images
        assert any(a.shape != b.shape or not torch.equal(a, b) for (a, _), (b, _) in zip(want[step], want[step - 1]))


# ---------------------------------------------------------------------------------------------------- teacher-forced networks
def check_ops_teacher_forced(net, ops, images, label, what=''):
    """one forward of images [B, 3, H, W] (float32 numpy) through net, then every op of `ops` (build_ops of net's plan)
    against kernel_refs.op_ref on the tensors the GPU actually fed it (each (tensor, column) has one producer:
    test_kernel_refs.py::test_every_tensor_column_is_written_by_one_op); every ratio is recorded under
    '<kind> (<label>)'.  -> ({kind: worst err / bound}, the head outputs of the forward as CUDA tensors)"""
    B = images.shape[0]
    fields = [t.clone() for t in net.forward(torch.from_numpy(images).cuda())]
    torch.cuda.synchronize()
    taps = {t: net.tap(t, B) for t in range(len(net.tensor_shapes))}
    heads = [t.cpu().numpy() for t in fields]
    worst = {}
    for i, o in enumerate(ops):
        kind, r = kr.op_ref(o, taps, heads, images, B)
        worst[kind] = max(worst.get(kind, 0.0), r)
        record(f'{kind} ({label})', r, f'{what} op {i}')
    return worst, fields


NETWORKS = [
    ('shufflenetv2k16', 'bins', True, 97, 129, 2),
    ('shufflenetv2k16', 'bins', False, 97, 129, 2),
    ('shufflenetv2k16', 'shuffle', False, 97, 129, 2),
    ('shufflenetv2k30-wholebody', 'bins', False, 129, 97, 2),
    ('resnet18', None, None, 161, 161, 1),
    ('resnet50', None, None, 129, 129, 2),
]


@pytest.mark.parametrize('name,layout,fuse,H,W,B', NETWORKS,
                         ids=['%s-%s-fuse%s' % (n[0], n[1], n[2]) for n in NETWORKS])
def test_teacher_forced_ops_of_real_networks(name, layout, fuse, H, W, B):
    """one forward, then every op against the float64 reference of the tensors the GPU actually fed it"""
    if name == 'shufflenetv2k30-wholebody':
        shell = net_oracle.make_shell('shufflenetv2k30', n_keypoints=133, n_connections=160, seed=3)
    else:
        shell = net_oracle.make_shell(name, seed=4)
    plan = network.plan_from_shell(shell)
    kw = {} if layout is None else {'layout': layout, 'fuse_dw': fuse}
    _, ops, _ = network.build_ops(plan, H, W, **kw)
    net = network.CompiledNet(plan, H, W, B, **kw)
    images = np.random.default_rng(9).standard_normal((B, 3, H, W)).astype(np.float32)
    worst, _ = check_ops_teacher_forced(net, ops, images, 'network', name)
    net.close()
    print(name, layout, fuse, {k: round(v, 3) for k, v in worst.items()})
