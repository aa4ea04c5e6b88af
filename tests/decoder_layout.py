"""Mirror of the shared-memory plan of the CUDA grow kernels (openpifpaf_b200/csrc/decoder.cu: `worker_bytes`,
`grow_fixed_bytes`, `plan_grow`, `LIST_SMEM_ENTRIES` and the greedy first-fit prefix of `grow_shared_init`).

The decoder picks its code path from this plan: how many warps a grow CTA runs (annotations grown at once), how many
CAF list entries it stages in shared memory, and which lists it reads from global memory instead.  The scale tests
use the mirror to choose inputs that reach every path; `test_decoder_layout.py` checks that the copied lines are
still those of decoder.cu."""
import numpy as np

LIST_SMEM_ENTRIES = 8192
GROW_MAX_WORKERS = 16

# list tiers of list_tiers(): (c, x_src, y_src) and (x_dst, y_dst, s_dst) staged / only (c, x_src, y_src) staged /
# everything read from global memory
STAGED, SRC_STAGED, GLOBAL = 0, 1, 2


def _align16(n):
    return (n + 15) & ~15


def worker_bytes(K, C):
    b = 24 * K + 24 * 2 * C + (4 + 2 * 4) * (2 * C + 2) + ((2 * C + 3) & ~3) + 32 * 4
    return _align16(b)


def grow_fixed_bytes(K, C):
    return _align16((8 * C + K + 1 + 2 * C + 2 * C + 8) * 4)


def plan_grow(K, C):
    """(workers, list_cap, ext_cap, smem) of decoder.cu's plan_grow"""
    budget, fixed = 200 * 1024, grow_fixed_bytes(K, C) + 64 * 4 + 256
    wb = worker_bytes(K, C)
    list_cap = LIST_SMEM_ENTRIES
    lists = 4 * 3 * list_cap
    if fixed + lists + 4 * wb > budget:
        list_cap = LIST_SMEM_ENTRIES // 2
        lists //= 2
    w = (budget - fixed - lists) // wb
    workers = max(1, min(GROW_MAX_WORKERS, w))
    used = fixed + lists + workers * wb
    ext = (budget - used) // (3 * 4) if used < budget else 0
    ext_cap = max(0, min(list_cap, ext // 32 * 32))
    return workers, list_cap, ext_cap, used + 4 * 3 * ext_cap


def list_tiers(counts, list_cap, ext_cap):
    """Tier of every CAF list of one image.  counts: list lengths in the decoder's order [C][2] (forward, backward)
    flattened; returns an int array of STAGED / SRC_STAGED / GLOBAL."""
    out = np.empty(len(counts), dtype=np.int64)
    run = 0
    for li, n in enumerate(int(c) for c in counts):
        if run + n <= list_cap:
            out[li] = STAGED if run + n <= ext_cap else SRC_STAGED
            run += n
        else:
            out[li] = GLOBAL
    return out


def oracle_list_counts(taps):
    """the list lengths of an oracle run (oracle.cifcaf.decode(..., taps=True)) in the decoder's order"""
    return np.stack([[len(f) for f in taps['fwd']], [len(b) for b in taps['bwd']]], axis=1).reshape(-1)


def synthetic_skeleton(K, C, seed, n_dup=4, n_rev=4):
    """1-based connection list of C pairs over K joints: a random spanning tree, then random extra pairs, with n_dup
    duplicated and n_rev reversed copies of earlier pairs at random places (the first-match rules of the decoder's
    edge lookup and frontier pair ids see them).  Only PCG64 doubles are drawn, like openpifpaf_b200.synth."""
    rng = np.random.Generator(np.random.PCG64(seed))
    pick = lambda n: int(rng.random() * n) % n      # noqa: E731
    order = list(range(K))
    for i in range(K - 1, 0, -1):
        j = pick(i + 1)
        order[i], order[j] = order[j], order[i]
    pairs = [(order[i], order[pick(i)]) for i in range(1, K)]
    while len(pairs) < C - n_dup - n_rev:
        a, b = pick(K), pick(K)
        if a != b:
            pairs.append((a, b))
    for k in range(n_dup + n_rev):
        a, b = pairs[pick(len(pairs))]
        pairs.insert(pick(len(pairs) + 1), (a, b) if k < n_dup else (b, a))
    return np.asarray(pairs, dtype=np.int64).reshape(C, 2) + 1


# ---- the CifCaf inputs of test_decoder_scale_gpu.py: name -> (synth.make_fields arguments, stride, tie quantisation)
# (quantisation: None, or 'levels' / 'binary' -- see tie_quantise)
SCALE_CASES = {
    'coco60_81x81_s8': (dict(workload='cocokp', h=81, w=81, n_people=60, seed=11), 8, None),
    'coco40_61x61': (dict(workload='cocokp', h=61, w=61, n_people=40, seed=12), 16, None),
    'wholebody8_41x41': (dict(workload='wholebody', h=41, w=41, n_people=8, seed=13), 16, None),
    'coco10_81x81_s8': (dict(workload='cocokp', h=81, w=81, n_people=10, seed=14), 8, None),
    'coco1_81x81_s8': (dict(workload='cocokp', h=81, w=81, n_people=1, seed=15), 8, None),
    'coco0_81x81_s8': (dict(workload='cocokp', h=81, w=81, n_people=0, seed=16, n_distractors=5), 8, None),
    'coco1_61x61': (dict(workload='cocokp', h=61, w=61, n_people=1, seed=17), 16, None),
    'wholebody1_41x41': (dict(workload='wholebody', h=41, w=41, n_people=1, seed=18), 16, None),
    'wholebody0_41x41': (dict(workload='wholebody', h=41, w=41, n_people=0, seed=19), 16, None),
    # narrow grow CTAs: K = 133 with 250 / 320 / 800 connections (4 workers; 5 workers and list_cap 4096; 1 worker)
    'skeleton250': (dict(workload='wholebody', h=41, w=41, n_people=10, seed=270, skeleton=250), 16, None),
    'skeleton320': (dict(workload='wholebody', h=41, w=41, n_people=10, seed=340, skeleton=320), 16, None),
    'skeleton800': (dict(workload='wholebody', h=41, w=41, n_people=6, seed=820, skeleton=800), 16, None),
    # exact seed-score ties
    'ties_saturated': (dict(workload='cocokp', h=81, w=81, n_people=60, seed=21), 8, 'saturate'),
    'ties_levels': (dict(workload='cocokp', h=81, w=81, n_people=60, seed=22), 8, 'levels'),
    'ties_uniform': (dict(workload='cocokp', h=61, w=61, n_people=30, seed=23), 16, 'binary'),
}


def tie_quantise(conf, how):
    """CIF / CifDet confidences with exact ties.  'saturate': the cores of the blobs at 1.0 (their CifHr saturates, so
    their seeds rescore to exactly 1.0); 'levels': every cell above 0.2 on one of 0.25 / 0.5 / 0.75 / 1.0 (low three
    key bytes equal); 'binary': 1.0 or 0.0 (every seed scores 1.0 without rescoring)"""
    c = conf.astype(np.float64)
    if how == 'saturate':
        out = np.where(c >= 0.5, 1.0, c)
    elif how == 'levels':
        out = np.where(c >= 0.2, np.ceil(c * 4.0) / 4.0, c)
    elif how == 'binary':
        out = np.where(c >= 0.3, 1.0, 0.0)
    else:
        raise ValueError(how)
    return out.astype(np.float32)


_fields_cache = {}


def scale_fields(name):
    """fields of SCALE_CASES[name] (cached; do not modify) and the case's stride and quantisation"""
    from openpifpaf_b200 import synth
    kw, stride, quant = SCALE_CASES[name]
    if name not in _fields_cache:
        kw = dict(kw)
        if isinstance(kw.get('skeleton'), int):
            kw['skeleton'] = synthetic_skeleton(133, kw['skeleton'], kw['skeleton'])
        f = synth.make_fields(**kw)
        if quant is not None:
            f['cif'][:, 1] = tie_quantise(f['cif'][:, 1], quant)
        _fields_cache[name] = f
    return _fields_cache[name], stride, quant
