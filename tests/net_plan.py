"""CPU mirror of the kernel-variant and resource plans that openpifpaf_b200/csrc/net.cu's host code makes at emit time:
the GEMM tile, weight residency, ring depth and epilogue of each k_gemm_wg op, the depthwise kernel, the fused
1x1 -> depthwise decision of plan_pw_dw and the ring plan of k_dw_gemm.  Pure Python; tests/test_net_plan.py pins the
copied source lines to net.cu and checks that the single-op GPU cases reach every plan the planner can make.

A GEMM op's plan is a Cell: route ('1x1', 'conv': implicit GEMM, 'heads'), epilogue (EPILOGUES), the k_gemm_wg
instantiation (NG column groups of 64, LASTW columns in the last group), weight residency and ring depth."""
from collections import namedtuple

BM, BK = 128, 64
NGROUP = 64
STG_BYTES = 8 * 16 * 33 * 4                  # CONSUMER_WARPS x 16 x STG_LD f32
GEMM_SMEM_BUDGET = 222 * 1024
MAX_STORE_MAPS = 8
PWDW_K = 32                                  # 1x1 input channels the k_pw_dw window carries
PW_DW_SMEM_LIMIT = 226 * 1024
WG_ROWS = 64

ROUTES = ('1x1', 'conv', 'heads')
EPILOGUES = ('tma plain', 'tma scatter', 'lane plain', 'lane residual', 'lane relu6', 'lane scatter',
             'shuffle src_tma', 'shuffle lane src', 'heads', 'heads upsampled')
INSTANTIATIONS = tuple((ng, lw) for ng in (1, 2, 3, 4) for lw in (16, 32, 48, 64))
Cell = namedtuple('Cell', 'route epilogue ng lastw resident stages')


def pad8(v):
    return (v + 7) // 8 * 8


def pad16(v):
    return (v + 15) // 16 * 16


def choose_block_n(n_out):
    """-> (block_n, n_blocks): the largest tile (<= 256 columns) whose padded work is within 10 % of the minimum"""
    np_ = pad16(n_out)
    cands = [(pad16((np_ + nb - 1) // nb), nb) for nb in range(1, np_ // 16 + 1)]
    cands = [(bn, nb) for bn, nb in cands if bn <= 256]
    min_cost = min(bn * nb for bn, nb in cands)
    for bn, nb in cands:
        if bn * nb * 100 <= min_cost * 110:
            return bn, nb
    return 16, np_ // 16


def gemm_smem_bytes(block_n, n_blocks, stages, shuffle, b_resident=False, num_k_blocks=0):
    b_stage = 0 if b_resident else block_n * BK * 2
    b_res = num_k_blocks * block_n * BK * 2 if b_resident else 0
    return (1024 + stages * (BM * BK * 2 + b_stage) + b_res + (2 * BM * block_n * 2 if shuffle else 0) +
            n_blocks * block_n * 5 + STG_BYTES + (2 * stages + 5) * 8 + 64)


def choose_stages(block_n, n_blocks, num_k_blocks, shuffle):
    stages = min(8, max(2, num_k_blocks * 2))
    while stages > 2 and gemm_smem_bytes(block_n, n_blocks, stages, shuffle) > GEMM_SMEM_BUDGET:
        stages -= 1
    return stages


def resident_stages(block_n, n_blocks, num_k_blocks, shuffle):
    if gemm_smem_bytes(block_n, n_blocks, 3, shuffle, True, num_k_blocks) > GEMM_SMEM_BUDGET:
        return 0
    stages = 8
    while gemm_smem_bytes(block_n, n_blocks, stages, shuffle, True, num_k_blocks) > GEMM_SMEM_BUDGET:
        stages -= 1
    return stages


def tile_groups(block_n):
    """-> (NG, LASTW) of the k_gemm_wg instantiation a block_n-column tile launches"""
    g = (block_n + NGROUP - 1) // NGROUP - 1
    return g + 1, block_n - g * NGROUP


def gemm_cell(route, k_cols, n_out, *, c_in=0, taps=1, residual=False, relu=0, shuffle=False, n_maps=0, up=1,
              tma_store=True, res_stages=0):
    """plan of one k_gemm_wg op.  route '1x1': k_cols input columns (plain, residual, shuffle, or a scatter into n_maps
    destination tensors when n_maps > 0); 'conv': c_in channels x taps (kernel^2); 'heads': n_out conv columns (fields
    x components x up^2).  tma_store / res_stages: PIFPAF_GEMM_TMA_STORE and PIFPAF_GEMM_RES_STAGES."""
    assert route in ROUTES
    block_n, n_blocks = choose_block_n(n_out)
    if route == 'conv':
        num_k_blocks = taps * ((c_in + BK - 1) // BK)
    else:
        num_k_blocks = (k_cols + BK - 1) // BK
        if res_stages > 0:                   # emit_gemm: narrower tiles until enough resident A stages fit
            np_ = pad16(n_out)
            st = resident_stages(block_n, n_blocks, num_k_blocks, False)
            while 0 < st < res_stages and block_n > 64:
                nb = n_blocks + 1
                bn = pad16((np_ + nb - 1) // nb)
                if bn < 64:
                    break
                n_blocks, block_n = nb, bn
                st = resident_stages(block_n, n_blocks, num_k_blocks, False)
    src_tma = False
    if route == 'heads':
        epilogue = 'heads upsampled' if up > 1 else 'heads'
    elif residual:
        epilogue = 'lane residual'
    elif route == 'conv':
        epilogue = 'lane relu6' if relu == 2 else 'lane plain'
    elif shuffle:
        src_tma = gemm_smem_bytes(block_n, n_blocks, 2, True) <= GEMM_SMEM_BUDGET
        epilogue = 'shuffle src_tma' if src_tma else 'shuffle lane src'
    elif n_maps > 0:
        epilogue = 'tma scatter' if tma_store and n_maps <= MAX_STORE_MAPS else 'lane scatter'
    elif relu == 2:
        epilogue = 'lane relu6'
    else:
        epilogue = 'tma plain' if tma_store else 'lane plain'
    res = resident_stages(block_n, n_blocks, num_k_blocks, src_tma) if route == '1x1' else 0
    stages = res if res > 0 else choose_stages(block_n, n_blocks, num_k_blocks, src_tma)
    ng, lastw = tile_groups(block_n)
    return Cell(route, epilogue, ng, lastw, res > 0, stages)


def op_cells(op):
    """the Cells of one op of network.build_ops (none for ops that are not k_gemm_wg launches)"""
    kind = op['kind']
    if kind == 'conv1x1':
        if 'pieces' in op:
            return [gemm_cell('1x1', op['k_cols'], op['n_out'], relu=op['relu'],
                              n_maps=len({p[2] for p in op['pieces']}))]
        return [gemm_cell('1x1', op['k_cols'], op['n_out'], relu=op['relu'], shuffle=op['shuffle_src'] >= 0)]
    if kind == 'conv':
        if op['kernel'] == 1 and op['stride'] == 1 and op['pad'] == 0:
            return [gemm_cell('1x1', op['c_in'], op['n_out'], relu=op['relu'], residual=op['residual'] >= 0)]
        return [gemm_cell('conv', 0, op['n_out'], c_in=op['c_in'], taps=op['kernel'] ** 2, relu=op['relu'],
                          residual=op['residual'] >= 0)]
    if kind == 'heads':
        up = op['upsample']
        n = sum(f * c for f, c in zip(op['n_fields'], op['n_comp'])) * up * up
        return [gemm_cell('heads', op['k_cols'], n, up=up)]
    return []


# ------------------------------------------------------------------------------------------------ depthwise
DW_S2_SMEM = 2 * 19 * 35 * 64 * 2 + 128      # DwS2::SMEM: two 19 x 35-pixel windows of 64 channels
DW_CBF_SMEM = 226 * 1024                     # DW_TMA[DW_K5_S2_CBF].smem


def dw_kernel(channels, kernel, stride, relu, dilation=1, gemm_impl=0, cbf=False):
    """the kernel a depthwise op launches (choose_dw_kernels): a DW_TMA entry ('DW_K5_S1', 'DW_K5_S2', 'DW_K5_S2_CBF',
    'DW_K3_S1', 'DW_K3_S2', 'DW_K5_S1_D2'), 'k_dwconv5' or 'k_dwconv'.  cbf: PIFPAF_DW_CBF"""
    tma = None
    if dilation == 2 and kernel == 5 and stride == 1 and relu != 2:
        tma = 'DW_K5_S1_D2'
    elif dilation == 1 and (kernel == 3 or (kernel == 5 and relu != 2)) and stride in (1, 2):
        tma = 'DW_K%d_S%d' % (kernel, stride)
    if tma and gemm_impl == 0:
        C = pad8(channels)
        if tma == 'DW_K5_S2' and cbf and (C // 8 + 7) // 8 > 1 and DW_S2_SMEM + 26 * C * 4 <= DW_CBF_SMEM:
            return 'DW_K5_S2_CBF'
        return tma
    if kernel == 5 and dilation == 1 and stride in (1, 2):
        return 'k_dwconv5'
    return 'k_dwconv'


# ------------------------------------------------------------------------------------------------ fused 1x1 -> depthwise
PWDW_IH, PWDW_IW = 7 * 2 + 5, 15 * 2 + 5    # PwDwS2: the input window of an 8 x 16 stride-2 output tile
PWDW_NPIX = PWDW_IH * PWDW_IW
PWDW_IN_BYTES = (PWDW_NPIX + WG_ROWS - 1) // WG_ROWS * WG_ROWS * 64
PWDW_MID_BYTES = PWDW_NPIX * 128


def pw_dw_smem_bytes(in_bytes, mid_bytes, cblks, c_dw):
    return 1024 + 2 * in_bytes + mid_bytes + cblks * 64 * (PWDW_K * 2 + 4) + c_dw * 26 * 4


def pw_dw_refusal(gemm, dw, in_pitch, others_touch_mid=False):
    """None when plan_pw_dw fuses the 1x1 op `gemm` with the depthwise op `dw` right after it, else the rule that
    refuses the pair.  gemm: a conv1x1 / conv op dict of network.build_ops, dw: a dwconv op dict; in_pitch: the
    channel pitch of the 1x1 input tensor; others_touch_mid: another op reads or writes the 1x1 output tensor."""
    if gemm['kind'] == 'conv1x1':
        k_cols, shuffle, residual, pieces = gemm['k_cols'], gemm['shuffle_src'] >= 0, False, 'pieces' in gemm
    elif gemm['kind'] == 'conv' and gemm['kernel'] == 1 and gemm['stride'] == 1 and gemm['pad'] == 0:
        k_cols, shuffle, residual, pieces = gemm['c_in'], False, gemm['residual'] >= 0, False
    else:
        return 'not a 1x1 GEMM'
    if dw['kind'] != 'dwconv' or dw_kernel(dw['channels'], dw['kernel'], dw['stride'], dw['relu'],
                                           dw.get('dilation', 1)) != 'DW_K5_S2':
        return 'depthwise is not the TMA 5x5 stride-2 kernel'
    if shuffle or pieces:
        return 'not a plain epilogue'
    if residual:
        return 'residual'
    if (k_cols + BK - 1) // BK != 1:
        return 'more than one K block'
    if gemm['in_off'] != 0:
        return 'input column offset'
    if gemm.get('out_off', 0) != 0:
        return 'output column offset'
    if gemm['relu'] == 2:
        return 'ReLU6'
    if dw['pad'] != 2:
        return 'depthwise pad'
    if dw['in'] != gemm['out']:
        return 'depthwise reads another tensor'
    if dw['in_off'] != 0:
        return 'depthwise input column offset'
    if in_pitch > PWDW_K:
        return 'input wider than PWDW_K'
    if others_touch_mid:
        return 'another op touches the intermediate'
    C = pad8(dw['channels'])
    if pw_dw_smem_bytes(PWDW_IN_BYTES, PWDW_MID_BYTES, (C // 8 + 7) // 8, C) > PW_DW_SMEM_LIMIT:
        return 'shared memory'
    return None


def fused_pairs(tensors, ops, fuse_pw_dw=True):
    """indices of the 1x1 ops plan_pw_dw elides (each fused into the depthwise op after it)"""
    if not fuse_pw_dw:
        return []
    touches = []
    for o in ops:
        t = {o.get('in', -1), o.get('out', -1), o.get('residual', -1), o.get('shuffle_src', -1)}
        t |= {p[2] for p in o.get('pieces', ())}
        touches.append(t)
    out = []
    for i in range(len(ops) - 1):
        g, d = ops[i], ops[i + 1]
        if g['kind'] not in ('conv1x1', 'conv'):
            continue
        mid = g['out']
        others = any(mid in touches[j] for j in range(len(ops)) if j not in (i, i + 1))
        if pw_dw_refusal(g, d, tensors[g['in']][2], others) is None:
            out.append(i)
    return out


# ------------------------------------------------------------------------------------------------ fused depthwise -> 1x1
def fused_rings(channels, n_out):
    """(window ring, B ring) depths that pifpaf_net_dw_conv1x1_scatter picks for a fused depthwise -> 1x1 op (k_dw_gemm):
    fused_smem_bytes, the candidate list {3,2},{2,2},{2,1},{1,1} and GEMM_SMEM_BUDGET; None if none fits"""
    C = pad8(channels)
    nb = (n_out + 191) // 192                    # FD_MAX_BLOCK_N = 3 x 64 columns per CTA
    bn = pad16((n_out + nb - 1) // nb)
    window = 12 * 20 * 64 * 2                    # DwTile<1, 8, 16, 4, 1>::BYTES: (8+4) x (16+4) pixels x 64 channels
    for ws, bs in ((3, 2), (2, 2), (2, 1), (1, 1)):
        size = (1024 + BM * BK * 2 + bs * bn * BK * 2 + ws * window + bn * nb * 5 + C * 26 * 4 + STG_BYTES
                + 2 * (ws + bs) * 8 + 64)
        if size <= GEMM_SMEM_BUDGET:
            return ws, bs
    return None
