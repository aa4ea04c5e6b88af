"""CPU: tests/net_plan.py against the net.cu lines it mirrors, and the single-op GPU cases against the plans net.cu's
host code can make.  A kernel variant, ring depth or epilogue that no single-op case reaches is tested only by
accident (inside a real network, at one size); these tests name every such hole."""
import os
import re
from collections import defaultdict

import net_plan as npl
from net_plan import gemm_cell
from openpifpaf_b200 import network

NET_CU = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'openpifpaf_b200', 'csrc', 'net.cu')

# the lines of net.cu that tests/net_plan.py copies (whitespace folded): change both together
MIRRORED = [
    # choose_block_n
    'for (int nb = 1; nb <= np / 16; nb++) { const int bn = pad16((np + nb - 1) / nb); if (bn > 256) continue; '
    'const long cost = (long)bn * nb; if (min_cost < 0 || cost < min_cost) min_cost = cost; }',
    'if ((long)bn * nb * 100 <= min_cost * 110) { *block_n = bn; *n_blocks = nb; return; } } '
    '*block_n = 16; *n_blocks = np / 16; }',
    # gemm_smem_bytes, choose_stages, resident_stages, plan_gemm_smem
    'const size_t b_stage = b_resident ? 0 : (size_t)block_n * BK * 2; '
    'const size_t b_res = b_resident ? (size_t)num_k_blocks * block_n * BK * 2 : 0; '
    'return 1024 + (size_t)stages * (BM * BK * 2 + b_stage) + b_res + (shuffle ? 2 * (size_t)BM * block_n * 2 : 0) + '
    '(size_t)n_blocks * block_n * 5 + STG_BYTES + (2 * stages + 5) * 8 + 64;',
    'int stages = std::min(8, std::max(2, num_k_blocks * 2)); '
    'while (stages > 2 && gemm_smem_bytes(block_n, n_blocks, stages, shuffle) > GEMM_SMEM_BUDGET) stages--;',
    'if (gemm_smem_bytes(block_n, n_blocks, 3, shuffle, true, num_k_blocks) > GEMM_SMEM_BUDGET) return 0; '
    'int stages = 8; '
    'while (gemm_smem_bytes(block_n, n_blocks, stages, shuffle, true, num_k_blocks) > GEMM_SMEM_BUDGET) stages--;',
    'const int res = g.conv_k == 0 && g.mode != MODE_HEADS ? '
    'resident_stages(g.block_n, g.n_blocks, g.num_k_blocks, src_tma) : 0;',
    'g.stages = res > 0 ? res : choose_stages(g.block_n, g.n_blocks, g.num_k_blocks, src_tma);',
    # PIFPAF_GEMM_RES_STAGES retiling (emit_gemm)
    'int st = resident_stages(block_n, n_blocks, num_k_blocks, false); '
    'while (st > 0 && st < net->gemm_res_stages && block_n > 64) { '
    'const int nb = n_blocks + 1, bn = pad16((np + nb - 1) / nb); if (bn < 64) break;',
    # epilogues: shuffle pass-through by TMA, TMA-store eligibility
    'g.src_tma = gemm_smem_bytes(g.block_n, g.n_blocks, 2, true) <= GEMM_SMEM_BUDGET ? 1 : 0;',
    'if (residual_tensor >= 0) return set_residual(net, g, residual_tensor, residual_col_off, to.h, to.w); '
    'if (net->gemm_tma_store && g.relu != ACT_RELU6) { g.tma_store = 1;',
    'if (net->gemm_tma_store && (int)map_tensor.size() <= MAX_STORE_MAPS) {',
    'inline int tile_groups(int block_n) { return (block_n + NGROUP - 1) / NGROUP - 1; }',
    'inline int tile_last(int block_n) { return (block_n - tile_groups(block_n) * NGROUP) / 16 - 1; }',
    # depthwise kernel selection (choose_dw_kernels)
    'const DwArgs& a = op.dw; const int kernel = a.kernel, stride = a.stride, relu = a.relu, dilation = op.dw_dil; '
    'if (dilation == 2 && kernel == 5 && stride == 1 && relu != ACT_RELU6) { op.dw_tma = &DW_TMA[DW_K5_S1_D2]; } '
    'else if (dilation == 1 && (kernel == 3 || (kernel == 5 && relu != ACT_RELU6)) && (stride == 1 || stride == 2)) { '
    'op.dw_tma = &DW_TMA[kernel == 3 ? (stride == 1 ? DW_K3_S1 : DW_K3_S2) : (stride == 1 ? DW_K5_S1 : DW_K5_S2)]; } '
    'if (op.dw_tma) op.smem = op.dw_tma->smem;',
    'const size_t smem_cf = op.smem + (size_t)26 * a.C8 * 8 * sizeof(float); '
    'if (op.dw_tma == &DW_TMA[DW_K5_S2] && net->dw_cbf && (a.C8 + 7) / 8 > 1 && '
    'smem_cf <= (size_t)DW_TMA[DW_K5_S2_CBF].smem) { op.dw_tma = &DW_TMA[DW_K5_S2_CBF]; op.smem = smem_cf; } '
    'if (kernel == 5 && dilation == 1 && (stride == 1 || stride == 2)) '
    'op.dw_simt5 = stride == 1 ? k_dwconv5<1> : k_dwconv5<2>; }',
    '{k_dwconv5_tma<2, DW2_TH, DW2_TW, 4, 2, true>, DwS2::THREADS, 226 * 1024,',
    'using DwS2 = DwTile<2, DW2_TH, DW2_TW, 4, 2>;',
    'static constexpr int SMEM = NSTAGE * BYTES + 128;',
    # plan_pw_dw and pw_dw_smem_bytes
    'if (gop.kind != OP_GEMM || dop.kind != OP_DW || !dop.dw_tma || d.kernel != 5 || d.stride != 2) continue;',
    'if (g.mode != MODE_PLAIN || g.conv_k != 0 || g.res != nullptr || g.num_k_blocks != 1 || g.a_col0 != 0 || '
    'g.out_col_off != 0 || g.relu == ACT_RELU6) continue;',
    'if (d.pad != 2 || d.in != g.out || d.in_col_off != 0) continue;',
    'if (tin.c > PWDW_K) continue;',
    'const int cblks = (d.C8 + 7) / 8; '
    'const size_t smem = pw_dw_smem_bytes(PwDwS2::IN_BYTES, PwDwS2::MID_BYTES, cblks, d.C8 * 8); '
    'if (!private_mid || smem > 226 * 1024) continue;',
    'return 1024 + 2 * (size_t)in_bytes + (size_t)mid_bytes + (size_t)cblks * 64 * (PWDW_K * 2 + 4) + '
    '(size_t)c_dw * 26 * 4;',
    'static constexpr int IH = (TH - 1) * S + 5, IW = (TW - 1) * S + 5;',
    'static constexpr int CHUNKS = (NPIX + WG_ROWS - 1) / WG_ROWS;',
    'static constexpr int IN_BYTES = CHUNKS * WG_ROWS * 64;',
    'static constexpr int MID_BYTES = NPIX * 128;',
    'constexpr int PWDW_TH = 8, PWDW_TW = 16, PWDW_BW = 2;',
    'constexpr int PWDW_K = 32;',
    # k_dw_gemm's ring plan (pifpaf_net_dw_conv1x1_scatter)
    'size_t fused_smem_bytes(int ws, int bs, int block_n, int n_pad, int c_dw) { return 1024 + (size_t)BM * BK * 2 + '
    '(size_t)bs * block_n * BK * 2 + (size_t)ws * DwTile<1, PH, PW, 4, 1>::BYTES + (size_t)n_pad * 5 + '
    '(size_t)c_dw * 26 * 4 + STG_BYTES + (size_t)(2 * (ws + bs)) * 8 + 64; }',
    'const int cand[][2] = {{3, 2}, {2, 2}, {2, 1}, {1, 1}};',
    'if (fused_smem_bytes(c[0], c[1], block_n, n_pad, C) <= GEMM_SMEM_BUDGET)',
    'const int n_blocks = (n_out + FD_MAX_BLOCK_N - 1) / FD_MAX_BLOCK_N;',
    'const int block_n = pad16((n_out + n_blocks - 1) / n_blocks);',
    'constexpr int FD_MAX_BLOCK_N = 3 * NGROUP;',
    # constants
    'constexpr size_t GEMM_SMEM_BUDGET = 222 * 1024;',
    'constexpr int MAX_STORE_MAPS = 8;',
    'constexpr int PH = 8, PW = 16;',
    'static constexpr int BYTES = IH * IW * 64 * 2;',
    'constexpr int STG_LD = 33;',
    'constexpr int STG_BYTES = CONSUMER_WARPS * 16 * STG_LD * 4;',
    'constexpr int CONSUMER_WARPS = 8;',
    'constexpr int BM = 128;',
    'constexpr int BK = 64;',
    'constexpr int WG_ROWS = 64;',
    'constexpr int NGROUP = 64;',
    'constexpr int DW1_TH = 8, DW1_TW = 16, DW2_TH = 8, DW2_TW = 16;',
]


def test_mirror_matches_net_cu():
    """the planner lines net_plan.py copies are still those of net.cu, and the mirror gives the plans net.cu's
    comments state (N = 368 -> 2 x 192; k_pw_dw fits 320 depthwise channels, not 328)"""
    flat = re.sub(r'\s+', ' ', open(NET_CU).read())
    for line in MIRRORED:
        assert line in flat, line
    assert npl.fused_rings(176, 176) == (3, 2) and npl.fused_rings(1024, 192) == (1, 1)
    assert npl.choose_block_n(368) == (192, 2)
    assert npl.PWDW_IN_BYTES == 45056 and npl.PWDW_MID_BYTES == 85120
    assert npl.pw_dw_smem_bytes(npl.PWDW_IN_BYTES, npl.PWDW_MID_BYTES, 5, 320) == 231296 <= npl.PW_DW_SMEM_LIMIT
    assert npl.pw_dw_smem_bytes(npl.PWDW_IN_BYTES, npl.PWDW_MID_BYTES, 6, 328) > npl.PW_DW_SMEM_LIMIT
    assert npl.DW_S2_SMEM == 170368


# ------------------------------------------------------------------------------------------------ reachable cells
def reachable_cells():
    """every Cell the planner makes over the admissible op domain (1x1 / heads K up to 32 K blocks, implicit convs of
    1..7 taps squared and up to 8 channel blocks, N up to 1024 columns; pad16(N) alone sets the tile)"""
    cells = set()
    ks = [8, 32] + [64 * i for i in range(1, 33)]
    ns = range(16, 1025, 16)
    for K in ks:
        for N in ns:
            for kw in ({}, {'tma_store': False}, {'residual': True}, {'relu': 2}, {'shuffle': True}, {'n_maps': 1},
                       {'n_maps': 1, 'tma_store': False}):
                cells.add(gemm_cell('1x1', K, N, **kw))
            if N >= 9 * 16:
                cells.add(gemm_cell('1x1', K, N, n_maps=9))
            cells.add(gemm_cell('heads', K, N))
            cells.add(gemm_cell('heads', K, N, up=2))
    for c_in in [3] + [64 * i for i in range(1, 9)]:
        for taps in (1, 9, 25, 49):
            for N in ns:
                for kw in ({}, {'residual': True}, {'relu': 2}):
                    cells.add(gemm_cell('conv', 0, N, c_in=c_in, taps=taps, **kw))
    return cells


def projections(cells):
    """(route, epilogue, NG, LASTW) and (route, resident, ring depth) of each cell"""
    return ({(c.route, c.epilogue, c.ng, c.lastw) for c in cells},
            {(c.route, c.resident, c.stages) for c in cells})


ROUTE_EPILOGUES = {'1x1': ('tma plain', 'tma scatter', 'lane plain', 'lane residual', 'lane relu6', 'lane scatter',
                           'shuffle src_tma', 'shuffle lane src'),
                   'conv': ('lane plain', 'lane residual', 'lane relu6'),
                   'heads': ('heads', 'heads upsampled')}

# why a cell of the full cross product never occurs
UNREACHABLE = {
    ('1x1', 'shuffle src_tma'): 'the pass-through double buffer of a 240- or 256-column tile does not fit',
    ('1x1', 'shuffle lane src'): 'tiles of <= 224 columns fit the pass-through double buffer (unless 4 blocks of 224)',
    ('1x1', 'resident'): 'a resident weight tile needs 3 A stages beside it: depth 2 is streaming only',
    ('conv', 'resident'): 'implicit convs always stream their weights',
    ('conv', 'streaming'): 'depth 2 K blocks, capped at 8: 1 K block -> 2 stages, more -> >= 4, which every tile fits',
    ('heads', 'resident'): 'the heads always stream their weights',
    ('heads', 'streaming'): 'depth 2 K blocks, capped at 8: 1 K block -> 2 stages, more -> >= 4, which every tile fits',
}


def test_reachable_cells_and_their_reasons():
    """every (route, epilogue) x instantiation and every (route, residency, depth) that the planner cannot make has a
    reason in UNREACHABLE"""
    by_inst, by_ring = projections(reachable_cells())
    missing = defaultdict(list)
    for route, eps in ROUTE_EPILOGUES.items():
        for ep in eps:
            for ng, lw in npl.INSTANTIATIONS:
                if (route, ep, ng, lw) not in by_inst:
                    missing[(route, ep)].append((ng, lw))
        for res in (True, False):
            for st in range(2, 9):
                if (route, res, st) not in by_ring:
                    missing[(route, 'resident' if res else 'streaming')].append(st)
    for k, v in sorted(missing.items()):
        print('unreachable', k, v, '--', UNREACHABLE.get(k))
    assert set(missing) <= set(UNREACHABLE), set(missing) - set(UNREACHABLE)


# ------------------------------------------------------------------------------------------------ GPU case lists
def _gemm_tuple_cells(K, N, shuffle, relu, both):
    cells = {gemm_cell('1x1', K, N, relu=relu, shuffle=shuffle)}
    if both:
        cells.add(gemm_cell('1x1', K, N, relu=relu, shuffle=shuffle, tma_store=False))
    return cells


def _scatter_tuple_cells(K, N, pieces, both, res_stages=0):
    n_maps = len({p[1] for p in pieces})
    cells = {gemm_cell('1x1', K, N, n_maps=n_maps, res_stages=res_stages)}
    if both:
        cells.add(gemm_cell('1x1', K, N, n_maps=n_maps, tma_store=False, res_stages=res_stages))
    return cells


def _conv_tuple_cells(c):
    _, _, c_in, k, stride, pad, N, _, res_col, relu = c[:10]
    if k == 1 and stride == 1 and pad == 0:
        return {gemm_cell('1x1', c_in, N, relu=relu, residual=res_col is not None)}
    return {gemm_cell('conv', 0, N, c_in=c_in, taps=k * k, relu=relu, residual=res_col is not None)}


def heads_columns(spec, up=1):
    """conv columns of a HEADS_CASES spec (test_kernels_gpu.heads_case)"""
    if spec == 'all':
        return 3 * 6 * up * up
    return sum(s[0] * len(network.head_ops(s[1], s[2], s[3], (True,) * s[2])) for s in spec) * up * up


def case_cells():
    """-> {Cell: [case ids]} of every single-op GPU case of k_gemm_wg"""
    import test_gemm_gpu as tg
    import test_gemm_store_gpu as ts
    import test_kernels_gpu as tk
    out = defaultdict(list)

    def add(cells, what):
        for c in cells:
            out[c].append(what)
    for c in tk.GEMM_CASES:
        add(_gemm_tuple_cells(c[2], c[3], c[6], c[7], False), 'kernels ' + tk.gemm_id(c))
    for c in ts.PLAIN_CASES:
        add(_gemm_tuple_cells(c[2], c[3], c[6], c[7], True), 'store ' + ts.plain_id(c))
    for c in tg.CASES:
        add(_gemm_tuple_cells(c[3], c[4], c[6], 1, False), 'gemm %s' % (c,))
    for c in tk.SCATTER_CASES:
        add(_scatter_tuple_cells(c[2], c[3], c[4], False), 'kernels ' + tk.scatter_id(c))
    for c in tk.SCATTER_CASES[3:5]:
        add(_scatter_tuple_cells(c[2], c[3], c[4], False, res_stages=5), 'res_stages ' + tk.scatter_id(c))
    for c in ts.SCATTER_CASES:
        add(_scatter_tuple_cells(c[2], c[3], c[4], True), 'store ' + ts.scatter_id(c))
    for c in tk.CONV_CASES:
        add(_conv_tuple_cells(c), 'kernels ' + tk.conv_id(c))
    for c in tk.HEADS_CASES:
        up = c[6] if len(c) > 6 else 1
        add({gemm_cell('heads', c[2], heads_columns(c[3], up), up=up)}, 'kernels ' + tk.heads_id(c))
    return out


def test_gpu_cases_reach_every_reachable_cell():
    """the single-op GPU cases reach every (route, epilogue, instantiation) and every (route, residency, ring depth)
    the planner can make; prints the table"""
    reached = case_cells()
    want_inst, want_ring = projections(reachable_cells())
    got_inst, got_ring = projections(reached)
    print()
    for route, eps in ROUTE_EPILOGUES.items():
        for ep in eps:
            row = ['%d/%-2d %s' % (ng, lw, 'x' if (route, ep, ng, lw) in got_inst else
                                   ('-' if (route, ep, ng, lw) in want_inst else ' '))
                   for ng, lw in npl.INSTANTIATIONS]
            print('%-5s %-16s %s' % (route, ep, ' '.join(row)))
        for res in (True, False):
            row = ['%d %s' % (st, 'x' if (route, res, st) in got_ring else ('-' if (route, res, st) in want_ring else ' '))
                   for st in range(2, 9)]
            print('%-5s %-16s %s' % (route, 'resident' if res else 'streaming', '  '.join(row)))
    assert got_inst <= want_inst and got_ring <= want_ring
    assert want_inst - got_inst == set(), sorted(want_inst - got_inst)
    assert want_ring - got_ring == set(), sorted(want_ring - got_ring)


def _product_plans():
    import det_models
    import mobilenetv2_models as mm
    heads_wb = ((133, 1, 1, 1), (160, 1, 2, 2))
    return [
        ('k16', network.random_plan('shufflenetv2k16', seed=0), True),
        ('k30', network.random_plan('shufflenetv2k30', seed=0), True),
        ('k30-wholebody', network.random_plan('shufflenetv2k30', heads=heads_wb, seed=0), True),
        ('k16-stride8', network.random_plan('shufflenetv2k16', seed=0, stage4_dilation=2), True),
        ('r18', network.random_resnet_plan('resnet18', seed=0), False),
        ('r50', network.random_resnet_plan('resnet50', seed=0), False),
        ('mobilenetv2', network.plan_from_shell(mm.make_pose_shell(seed=0)), False),
        ('cocodet', network.plan_from_shell(det_models.make_variant_shell('cocodet', seed=0)), False),
    ]


def product_ops():
    """(name, layout, fuse_dw, tensors, ops) of the shipped plans at 641 x 641"""
    for name, plan, shufflenet in _product_plans():
        for layout, fuse in ((('bins', True), ('bins', False), ('shuffle', True), ('shuffle', False)) if shufflenet
                             else ((None, None),)):
            kw = {} if layout is None else {'layout': layout, 'fuse_dw': fuse}
            tensors, ops, _ = network.build_ops(plan, 641, 641, **kw)
            yield name, layout, fuse, tensors, ops


def test_product_cells_are_reachable_and_reached():
    """every GEMM plan of the shipped networks (641 px, both layouts, fuse_dw on and off) is a plan the planner can make,
    and a single-op GPU case runs that very plan: route, epilogue, instantiation, residency and ring depth together.
    The 1x1s that plan_pw_dw fuses into k_pw_dw launch no k_gemm_wg and are left out."""
    want_inst, want_ring = projections(reachable_cells())
    reached = case_cells()
    seen, missing = set(), {}
    for name, layout, fuse, tensors, ops in product_ops():
        elided = set(npl.fused_pairs(tensors, ops))
        for i, o in enumerate(ops):
            if i in elided:
                continue
            for c in npl.op_cells(o):
                seen.add(c)
                assert (c.route, c.epilogue, c.ng, c.lastw) in want_inst, (name, layout, fuse, c)
                assert (c.route, c.resident, c.stages) in want_ring, (name, layout, fuse, c)
                if c not in reached:
                    missing.setdefault(c, (name, layout, fuse, o['kind'], o.get('k_cols', o.get('c_in')), o['n_out']))
    print('\n%d distinct GEMM plans in the shipped networks' % len(seen))
    assert not missing, '\n'.join('%s: %s' % kv for kv in sorted(missing.items()))


# ------------------------------------------------------------------------------------------------ depthwise and k_pw_dw
def test_depthwise_cases_name_their_kernels():
    """the depthwise cases of test_kernels_gpu.py are labelled with the kernel net.cu launches for them, and reach
    every one: the TMA entries, k_dwconv5 and k_dwconv at stride 1 and 2"""
    import test_kernels_gpu as tk
    reached = set()
    for c in tk.DW5_CASES:
        for impl in (0, 1):
            reached.add((npl.dw_kernel(c[2], c[3], c[4], c[8], 1, impl), c[4]))
    for c in tk.DWK_CASES:
        dil, impl = c[11:13] if len(c) > 11 else (1, 0)
        kern = npl.dw_kernel(c[2], c[3], c[4], c[8], dil, impl)
        assert tk.dw_label(c[2], c[3], c[4], c[8], dil, impl).endswith(' ' + kern)
        reached.add((kern, c[4]))
    print(sorted(reached))
    assert {('DW_K5_S1', 1), ('DW_K5_S2', 2), ('DW_K3_S1', 1), ('DW_K3_S2', 2), ('k_dwconv5', 1), ('k_dwconv5', 2),
            ('k_dwconv', 1), ('k_dwconv', 2)} <= reached
    # the SM-limit sweep's depthwise cases: a name saying 'generic' runs k_dwconv, 'simt' k_dwconv5, any other a
    # DW_TMA entry -- as the kernel label the case's factory builds from the mirror says
    for name, (factory, impl) in tk.SCHEDULE_CASES.items():
        if not name.startswith('dwconv'):
            continue
        kern = factory()[2].kind.split()[-1]
        if 'generic' in name:
            assert kern == 'k_dwconv', (name, kern)
        elif 'simt' in name:
            assert kern == 'k_dwconv5' and impl == 1, (name, kern)
        else:
            assert kern.startswith('DW_') and impl == 0, (name, kern)


def test_pw_dw_cases_cover_the_admissible_domain_and_every_rule():
    """k_pw_dw's cases reach 1..5 channel blocks, input pitches 16 and 32, K = 8 / 16 / 24 / 32, every activation
    pair and a depthwise narrower than the 1x1; each refusal rule of plan_pw_dw has a pair that it alone refuses"""
    import test_pw_dw_gpu as tp
    cblks, pitches, ks, relus, narrow = set(), set(), set(), set(), False
    for H, W, K, N, C, pitch, relu1, relu2, batch, mb in tp.PAIR_CASES:
        assert batch < mb
        cblks.add((npl.pad8(C) // 8 + 7) // 8)
        pitches.add(pitch)
        ks.add(K)
        relus.add((relu1, relu2))
        narrow |= C < N
    assert cblks == {1, 2, 3, 4, 5} and pitches == {16, 32} and ks == {8, 16, 24, 32} and narrow
    assert relus == {(0, 0), (0, 1), (1, 0), (1, 1)}
    assert max(c[4] for c in tp.PAIR_CASES) == 320     # the widest depthwise that fits (328 does not: RULE_CASES)
    reasons = {tp.rule_pair(r).refusal() for r in tp.RULE_CASES}
    src = open(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'net_plan.py')).read()
    rules = set(re.findall(r"return '([^']+)'", src[src.index('def pw_dw_refusal'):src.index('def fused_pairs')]))
    # the GEMM kinds net_plan rejects before the rules (not a 1x1, shuffle / scatter epilogue) and the one that
    # cannot occur alone (a 1x1 reading more than one K block also reads more than PWDW_K columns)
    assert rules - reasons == {'not a 1x1 GEMM', 'not a plain epilogue', 'more than one K block',
                               'depthwise reads another tensor'}, rules - reasons

