"""CPU: tests/decoder_layout.py copies the grow plan of decoder.cu, and the inputs of test_decoder_scale_gpu.py still
reach every path of that plan (list tiers, grow CTA widths, staging sizes)."""
import os
import re

import numpy as np

import decoder_layout as L
from oracle import cifcaf as oc

DECODER_CU = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'openpifpaf_b200', 'csrc',
                          'decoder.cu')


def test_grow_plan_mirror_matches_decoder_cu():
    """the lines decoder_layout copies are still those of decoder.cu (change both together)"""
    flat = re.sub(r'\s+', ' ', open(DECODER_CU).read())
    for line in [
        'constexpr int LIST_SMEM_ENTRIES = 8192;',
        'constexpr int GROW_MAX_WORKERS = 16;',
        'struct WJoint { double v; float x, y, s; int pad; };',
        'size_t b = sizeof(WJoint) * (size_t)K + sizeof(WJoint) * 2 * (size_t)C + (sizeof(float) + 2 * sizeof(int)) * '
        '(2 * (size_t)C + 2) + ((2 * (size_t)C + 3) & ~(size_t)3) + 32 * sizeof(int); return (b + 15) & ~(size_t)15;',
        'return (((size_t)(8 * C + K + 1 + 2 * C + 2 * C + 8) * sizeof(int)) + 15) & ~(size_t)15;',
        'const size_t budget = 200 * 1024, fixed = grow_fixed_bytes(K, C) + 64 * sizeof(int) + 256;',
        'l.list_cap = LIST_SMEM_ENTRIES; size_t lists = sizeof(float) * 3 * (size_t)l.list_cap;',
        'if (fixed + lists + 4 * wb > budget) { l.list_cap = LIST_SMEM_ENTRIES / 2; lists /= 2; }',
        'long w = (long)((budget - fixed - lists) / wb);',
        'l.workers = (int)std::max(1L, std::min((long)GROW_MAX_WORKERS, w));',
        'const size_t used = fixed + lists + (size_t)l.workers * wb;',
        'long ext = used < budget ? (long)((budget - used) / (3 * sizeof(float))) : 0;',
        'l.ext_cap = (int)std::max(0L, std::min((long)l.list_cap, ext / 32 * 32));',
        'l.smem = used + sizeof(float) * 3 * (size_t)l.ext_cap;',
        # greedy first-fit prefix of grow_shared_init, and the tier tests of warp_connection_value
        'if (run + n <= list_cap) { s_loff[li] = run; run += n; } else s_loff[li] = -1;',
        'if (off + n <= ext_cap) {',
        'const bool fe = of >= 0 && of + nf <= g.ext_cap;',
        'const bool be = ob >= 0 && ob + nb <= g.ext_cap;',
        # list order: [C][2] (forward, backward) per image
        'const int lif = caf_i * 2 + (forward ? 0 : 1), lib = caf_i * 2 + (forward ? 1 : 0);',
    ]:
        assert line in flat, line
    assert L.plan_grow(17, 19)[:3] == (16, 8192, 6112)          # COCO
    assert L.plan_grow(133, 160)[:3] == (6, 8192, 544)          # WholeBody


def test_list_tiers_first_fit():
    t = L.list_tiers([100, 300, 50, 0, 10], list_cap=400, ext_cap=128)
    assert t.tolist() == [L.STAGED, L.SRC_STAGED, L.GLOBAL, L.SRC_STAGED, L.GLOBAL]


def test_scale_cases_reach_every_grow_path():
    """every tier of CAF list, grow CTAs of 16, 6, 4 or 5 and 1 warps, both staging sizes"""
    tiers, workers, caps = set(), set(), set()
    for name in L.SCALE_CASES:
        f, stride, quant = L.scale_fields(name)
        K, C = f['n_keypoints'], f['skeleton'].shape[0]
        p = oc.default_params(seed_sort_stable=1, seeds_ablation_no_rescore=int(quant in ('levels', 'binary')))
        _, _, ot = oc.decode(f['cif'], stride, f['caf'], stride, f['skeleton'], K, params=p, taps=True)
        w, list_cap, ext_cap, _ = L.plan_grow(K, C)
        t = L.list_tiers(L.oracle_list_counts(ot), list_cap, ext_cap)
        tiers |= set(t.tolist())
        workers.add(w)
        caps.add(list_cap)
        if (t == L.GLOBAL).any():
            assert L.oracle_list_counts(ot).sum() > list_cap
    assert tiers == {L.STAGED, L.SRC_STAGED, L.GLOBAL}
    assert {16, 6, 1} <= workers and workers & {4, 5}
    assert caps == {8192, 4096}


def test_synthetic_skeletons():
    for C in (250, 320, 800):
        sk = L.synthetic_skeleton(133, C, C)
        assert sk.shape == (C, 2) and sk.min() == 1 and sk.max() == 133 and (sk[:, 0] != sk[:, 1]).all()
        pairs = [tuple(p) for p in sk.tolist()]
        assert len(set(pairs)) < len(pairs) and any((b, a) in pairs for a, b in pairs)
        # the spanning tree connects every joint
        seen, todo = {1}, [1]
        while todo:
            j = todo.pop()
            for a, b in pairs:
                for u, v in ((a, b), (b, a)):
                    if u == j and v not in seen:
                        seen.add(v)
                        todo.append(v)
        assert len(seen) == 133
        np.testing.assert_array_equal(sk, L.synthetic_skeleton(133, C, C))
