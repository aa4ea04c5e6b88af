"""GPU: the TMA-store epilogue of k_gemm_wg (plain GEMMs without a residual and scatter GEMMs; on unless
PIFPAF_GEMM_TMA_STORE=0) against the float64 bound of tests/kernel_refs.py and bit for bit against the per-lane store
epilogue it replaces.

Single-op cases reuse the harness of test_kernels_gpu.py: a net whose max_batch exceeds the batch, random bf16 inputs
in every column, every output starting as the sentinel, which must survive outside the op's columns and in images
past the batch.  Tile widths: block_n = pad16(N) for N <= 256, so the plain cases below reach every (column groups,
last group width) instantiation, 1-4 groups of 16/32/48/64 columns."""
import numpy as np
import pytest
import torch

from openpifpaf_b200 import network
from test_kernels_gpu import gemm_case, n_sm, scatter_case

pytestmark = pytest.mark.gpu


def run_both(case, emit, batch, monkeypatch, **kw):
    """-> (taps with the TMA-store epilogue, taps with the per-lane store epilogue)"""
    monkeypatch.setenv('PIFPAF_GEMM_TMA_STORE', '1')
    tma, _ = case.run(emit, batch, **kw)
    monkeypatch.setenv('PIFPAF_GEMM_TMA_STORE', '0')
    lane, _ = case.run(emit, batch, **kw)
    monkeypatch.delenv('PIFPAF_GEMM_TMA_STORE')
    return tma, lane


def assert_same(a, b, what):
    for t in b:
        assert np.array_equal(a[t], b[t]), (what, t)


# (h, w, K, N, in_off, out_off, shuffle, relu, batch, max_batch); 99 / 91 / 144 / 117 rows per image: the last M tile
# of every case is partial.  N = bn - 10 leaves pad8(N) < block_n (a half-written last box), N = bn - 4 fills it.
PLAIN_CASES = [
    (9, 11, 40, 16, 0, 0, False, 1, 2, 3),          # 1 group: 16
    (9, 11, 72, 22, 8, 16, False, 0, 2, 3),         # 1 group: 32, pad8(N) = 24
    (13, 7, 64, 44, 0, 32, False, 1, 1, 2),         # 1 group: 48
    (13, 9, 130, 64, 0, 0, False, 0, 3, 4),         # 1 group: 64, K tail
    (12, 12, 176, 70, 0, 16, False, 1, 2, 3),       # 2 groups: 64 + 16
    (12, 12, 200, 92, 8, 0, False, 0, 2, 3),        # 64 + 32
    (9, 11, 96, 108, 0, 0, False, 1, 2, 3),         # 64 + 48
    (9, 11, 352, 124, 0, 16, False, 0, 1, 3),       # 64 + 64
    (13, 9, 176, 140, 0, 0, False, 1, 2, 3),        # 3 groups: 128 + 16
    (13, 9, 192, 150, 16, 0, False, 0, 2, 3),       # 128 + 32
    (12, 12, 174, 174, 176, 0, False, 0, 1, 3),     # 128 + 48 (the stage-2 pw1 width)
    (12, 12, 384, 188, 0, 0, False, 1, 2, 3),       # 128 + 64
    (13, 9, 416, 208, 0, 0, False, 1, 2, 3),        # 4 groups: 192 + 16
    (9, 11, 352, 214, 0, 16, False, 0, 2, 3),       # 192 + 32
    (9, 11, 64, 236, 0, 0, False, 1, 3, 4),         # 192 + 48
    (13, 9, 256, 256, 0, 0, False, 1, 2, 4),        # 192 + 64
    (41, 41, 1392, 240, 0, 32, False, 0, 1, 2),     # streaming weights
    (64, 64, 32, 174, 0, 0, False, 1, 3, 4),        # K = 32 (one half-filled K block), many tiles per CTA
    (41, 41, 704, 696, 0, 0, False, 1, 2, 3),       # 3 column blocks, tensor-bound stage-4 shape
    # the plain plans of the shipped networks' 1x1s (tests/test_net_plan.py lists them)
    (9, 11, 512, 128, 0, 0, False, 1, 2, 3),        # 2 x 64, resident 4
    (9, 11, 256, 128, 0, 16, False, 0, 2, 3),       # 2 x 64, resident 8
    (9, 11, 576, 160, 0, 0, False, 0, 2, 3),        # 3 x 64 - 32, streaming 5
    (9, 11, 400, 348, 0, 0, False, 1, 2, 3),        # 176 x 2, resident 3
    (9, 11, 208, 174, 0, 0, False, 1, 2, 3),        # 176, resident 7
    (9, 11, 272, 256, 0, 0, False, 1, 2, 3),        # 256, streaming 4
    (9, 11, 32, 256, 0, 0, False, 1, 2, 3),         # 256, resident 8
]


def plain_id(c):
    return 'hw%dx%d-K%d-N%d-in%d-out%d-relu%d-B%dof%d' % (c[:6] + c[7:])


@pytest.mark.parametrize('c', PLAIN_CASES, ids=plain_id)
def test_plain_tma_store_matches_float64_and_lane_stores(c, monkeypatch):
    case, emit, chk = gemm_case(*c)
    tma, lane = run_both(case, emit, c[8], monkeypatch)
    chk.kind = 'gemm plain tma-store'
    print(plain_id(c), '%.3f' % chk.verify(tma, plain_id(c)))
    assert_same(tma, lane, plain_id(c))


# (h, w, K, n_out, pieces [(count, dest, col)], dest widths, relu, batch, max_batch)
SCATTER_CASES = [
    (9, 11, 72, 48, [(48, 0, 16)], [64], 1, 2, 3),                                              # 1 piece
    (9, 11, 72, 48, [(16, 0, 16), (16, 1, 0), (16, 2, 32)], [48, 32, 64], 0, 2, 3),
    # the stage-1 layout: a 16-channel hole in front of the stride-2 depthwise input, other pitches around it
    (17, 13, 176, 176, [(32, 0, 0), (64, 1, 16), (48, 0, 48), (32, 2, 0)], [96, 96, 32], 1, 1, 2),
    (17, 13, 1392, 368, [(176, 0, 32), (192, 1, 0)], [224, 208], 1, 2, 3),                     # streaming
    # 8 pieces into 8 tensors (every store map), pitches 16 .. 128
    (41, 43, 352, 176, [(16, 0, 0), (32, 1, 16), (16, 2, 0), (16, 3, 32), (32, 4, 0), (16, 5, 64),
                        (32, 6, 16), (16, 7, 0)], [16, 48, 32, 64, 32, 128, 48, 16], 1, 2, 3),
    # 9 destination tensors: more than the store maps, the per-lane epilogue
    (33, 35, 352, 144, [(16, i, 0) for i in range(9)], [16] * 9, 0, 3, 4),
    (33, 35, 352, 192, [(192, 0, 0)], [208], 1, 3, 4),
    # 9 destination tensors in a 4-group tile (block_n = 256)
    (13, 9, 176, 256, [(16, i, 16 * ((i + 1) % 2)) for i in range(8)] + [(128, 8, 0)], [32, 16] * 4 + [128], 1, 2, 3),
] + [
    # every instantiation (block_n = N = 16 .. 256): a 16-column piece at a column offset, the rest in another tensor
    (9, 11, 72, n, [(16, 0, 16)] + ([(n - 16, 1, 0)] if n > 16 else []), [48, n + 16], n // 16 % 2, 2, 3)
    for n in range(16, 257, 16)
] + [
    # the scatter plans of the shipped ShuffleNetV2K stage GEMMs (tests/test_net_plan.py lists them)
    (9, 11, 256, 304, [(32, i, 0) for i in range(7)] + [(80, 7, 16)], [32] * 7 + [96], 1, 2, 3),   # 3 x 64 + 32, resident 7
    (9, 11, 512, 528, [(64, i, 16) for i in range(6)] + [(144, 6, 0)], [80] * 6 + [144], 0, 2, 3),  # 176 x 3, streaming 5
    (9, 11, 352, 400, [(48, i, 0) for i in range(6)] + [(112, 6, 16)], [48] * 6 + [128], 1, 2, 3),  # 208 x 2, streaming 4
    (9, 11, 176, 208, [(48, 0, 0), (48, 1, 16), (64, 2, 0), (48, 3, 32)], [48, 64, 64, 80], 1, 2, 3),   # resident 7
    (9, 11, 704, 704, [(224, 0, 0), (240, 1, 16), (240, 2, 0)], [224, 256, 240], 1, 2, 3),  # 240 x 3, streaming 4
    (9, 11, 512, 512, [(256, 0, 0), (256, 1, 16)], [256, 272], 0, 2, 3),                   # 256 x 2, streaming 4
    (9, 11, 256, 256, [(128, 0, 0), (128, 1, 0)], [128, 144], 1, 2, 3),                    # 256, resident 4
]


def scatter_id(c):
    return 'hw%dx%d-K%d-N%d-%dpieces-relu%d-B%dof%d' % (c[:4] + (len(c[4]),) + c[6:])


@pytest.mark.parametrize('c', SCATTER_CASES, ids=scatter_id)
def test_scatter_tma_store_matches_float64_and_lane_stores(c, monkeypatch):
    case, emit, chk = scatter_case(*c)
    tma, lane = run_both(case, emit, c[7], monkeypatch)
    chk.kind = 'gemm scatter tma-store'
    print(scatter_id(c), '%.3f' % chk.verify(tma, scatter_id(c)))
    assert_same(tma, lane, scatter_id(c))


SCHEDULE_CASES = {
    'plain resident': lambda: gemm_case(64, 64, 352, 176, 0, 0, False, 0, 3, 4),
    'plain K32': lambda: gemm_case(64, 64, 32, 174, 0, 0, False, 1, 3, 4),
    'plain streaming': lambda: gemm_case(41, 41, 1392, 240, 0, 32, False, 0, 2, 3),
    'scatter resident': lambda: scatter_case(*SCATTER_CASES[6]),
    'scatter 8 maps': lambda: scatter_case(*SCATTER_CASES[4]),
    'scatter 4 groups streaming': lambda: scatter_case(41, 43, 704, 704, [(224, 0, 0), (240, 1, 16), (240, 2, 0)],
                                                       [224, 256, 240], 1, 2, 3),
    'plain 3 groups resident 7': lambda: gemm_case(64, 64, 208, 174, 0, 0, False, 1, 3, 4),
}


@pytest.mark.parametrize('name', list(SCHEDULE_CASES))
def test_tma_store_sm_limit_is_bitwise_invariant(name, monkeypatch):
    """persistent grids capped at 1, 7 and n_sm - 4 SMs: every CTA walks more tiles, the output chunk buffers and
    bulk groups cycle across tiles; the outputs equal the per-lane store epilogue's bit for bit"""
    case, emit, chk = SCHEDULE_CASES[name]()
    batch = case.mb - 1
    _, want = run_both(case, emit, batch, monkeypatch)
    monkeypatch.setenv('PIFPAF_GEMM_TMA_STORE', '1')
    for lim in (1, 7, n_sm() - 4):
        taps, _ = case.run(emit, batch, sm_limit=lim)
        assert_same(taps, want, (name, lim))
    chk.verify(taps, name)


def forward_fields(plan, H, W, mb, x, tma, pdl, monkeypatch):
    monkeypatch.setenv('PIFPAF_GEMM_TMA_STORE', tma)
    monkeypatch.setenv('PIFPAF_PDL', pdl)
    net = network.CompiledNet(plan, H, W, mb)
    try:
        return [t.clone() for t in net.forward(x)]
    finally:
        net.close()


def test_network_pdl_and_store_paths_bitwise_equal(monkeypatch):
    """a k16 net, 3 of 4 images: PDL on and off, TMA stores on and off -- four times the same fields"""
    plan = network.random_plan('shufflenetv2k16', seed=3)
    x = torch.randn(3, 3, 129, 161, generator=torch.Generator().manual_seed(4)).cuda()
    want = forward_fields(plan, 129, 161, 4, x, '0', '1', monkeypatch)
    for tma, pdl in (('1', '1'), ('1', '0'), ('0', '0')):
        got = forward_fields(plan, 129, 161, 4, x, tma, pdl, monkeypatch)
        for a, b in zip(got, want):
            assert torch.isfinite(a).all() and torch.equal(a, b), (tma, pdl)


def test_bench_sized_network_store_paths_bitwise_equal(monkeypatch):
    """the k16 network at the benchmark's size (64 images of 641 x 641): the same fields with TMA stores on and off"""
    plan = network.random_plan('shufflenetv2k16', seed=0)
    x = torch.randn(64, 3, 641, 641, generator=torch.Generator().manual_seed(1)).cuda()
    want = forward_fields(plan, 641, 641, 64, x, '0', '1', monkeypatch)
    got = forward_fields(plan, 641, 641, 64, x, '1', '1', monkeypatch)
    for a, b in zip(got, want):
        assert torch.isfinite(a).all() and torch.equal(a, b)
