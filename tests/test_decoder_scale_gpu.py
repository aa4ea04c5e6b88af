"""GPU: the CUDA decoders at crowd scale, against the plain-C oracle.

The grow kernels choose their code path from the workload (tests/decoder_layout.py mirrors the plan): CAF lists beyond
the shared-memory staging area are read from global memory, wide skeletons shrink the grow CTA to fewer warps and a
smaller staging area, and packed results beyond the 512 KB fetch prefix take a second copy.  Every case here is built
to reach one of those paths (test_decoder_layout.py checks on the CPU that they still do), and every output is compared
with the oracle: CifHr, seeds and CAF lists bit for bit, annotations within the parity tolerances, ids equal."""
import numpy as np
import pytest
import torch

import decoder_layout as L
import helpers
from openpifpaf_b200 import decoder, synth
from oracle import cifcaf as oc

pytestmark = pytest.mark.gpu


def configure(**statics):
    C = decoder.CifCaf
    C.set_greedy(bool(statics.get('greedy', False)))
    C.set_force_complete(bool(statics.get('force_complete', False)))
    C.set_reverse_match(bool(statics.get('reverse_match', True)))
    decoder.CifSeeds.set_ablation_no_rescore(bool(statics.get('seeds_ablation_no_rescore', False)))


@pytest.fixture(autouse=True)
def reset_statics():
    yield
    configure()
    decoder.CifDet.set_max_detections_before_nms(120)


def oracle(f, stride, quant=None, **params):
    """oracle annotations, ids and stage taps, with the decoder statics of `params` and `quant`"""
    params.setdefault('seeds_ablation_no_rescore', int(quant in ('levels', 'binary')))
    p = oc.default_params(seed_sort_stable=1, **params)
    return oc.decode(f['cif'], stride, f['caf'], stride, f['skeleton'], f['n_keypoints'], params=p, taps=True)


def assert_stages_equal(d, ot, image=0, lists=True):
    np.testing.assert_array_equal(d.tap_cifhr(image).numpy(), ot['cifhr'])
    sf, sv = d.tap_seeds(image)
    np.testing.assert_array_equal(sf.numpy(), ot['seeds_f'])
    np.testing.assert_array_equal(sv.numpy(), ot['seeds_vxys'])
    if lists:
        fw, bw = d.tap_caf(image)
        for c, (a, b) in enumerate(zip(fw + bw, ot['fwd'] + ot['bwd'])):
            np.testing.assert_array_equal(a.numpy(), b, err_msg=f'CAF list {c}')


def single_decode(name, **statics):
    """decode of one SCALE_CASES input on a fresh handle, checked stage by stage against the oracle"""
    f, stride, quant = L.scale_fields(name)
    configure(seeds_ablation_no_rescore=quant in ('levels', 'binary'), **statics)
    oa, oi, ot = oracle(f, stride, quant, **{k: int(v) for k, v in statics.items()})
    d = decoder.CifCaf(f['n_keypoints'], torch.from_numpy(f['skeleton']))
    ga, gi = d.call(torch.from_numpy(f['cif']), stride, torch.from_numpy(f['caf']), stride)
    assert_stages_equal(d, ot, lists=not statics.get('force_complete'))
    helpers.assert_annotations_close(ga.numpy(), oa, name)
    np.testing.assert_array_equal(gi.numpy(), oi)
    return d, ot, ga


# ---- 1. CAF lists in every staging tier

@pytest.mark.parametrize('name', ['coco60_81x81_s8', 'coco40_61x61', 'wholebody8_41x41'])
def test_caf_lists_beyond_shared_memory(name):
    f, _, _ = L.scale_fields(name)
    d, ot, _ = single_decode(name)
    counts = L.oracle_list_counts(ot)
    _, list_cap, ext_cap, _ = L.plan_grow(f['n_keypoints'], f['skeleton'].shape[0])
    tiers = L.list_tiers(counts, list_cap, ext_cap)
    assert (tiers == L.GLOBAL).any() and (tiers == L.SRC_STAGED).any()
    entries = d.last_stats()['caf_entries']
    assert entries == counts.sum() and entries > list_cap


@pytest.mark.parametrize('statics', [dict(greedy=True), dict(force_complete=True), dict(reverse_match=False)],
                         ids=['greedy', 'force_complete', 'no_reverse_match'])
def test_caf_lists_beyond_shared_memory_other_modes(statics):
    single_decode('coco60_81x81_s8', **statics)


# ---- 2. grow CTAs of 4, 5 and 1 warps (wide synthetic skeletons on K = 133)

@pytest.mark.parametrize('name,workers,list_cap', [('skeleton250', 4, 8192), ('skeleton320', 5, 4096),
                                                   ('skeleton800', 1, 4096)])
def test_narrow_grow_ctas(name, workers, list_cap):
    f, _, _ = L.scale_fields(name)
    assert L.plan_grow(133, f['skeleton'].shape[0])[:2] == (workers, list_cap)
    sk = f['skeleton']
    pairs = [tuple(p) for p in sk.tolist()]
    assert len(set(pairs)) < len(pairs) and any((b, a) in pairs for a, b in pairs)    # duplicated + reversed pairs
    d, ot, ga = single_decode(name)
    st = d.last_stats()
    assert len(ga) > workers and st['grow_seeds_grown'] > workers
    if workers > 1:
        assert st['grow_seeds_grown'] > st['grow_rounds']      # rounds grew several annotations at once


def test_oracle_equals_reference_on_a_wide_synthetic_skeleton():
    if not oc.ref_available():
        pytest.skip('oracle/_ref/refcpp.so not built')
    f, stride, _ = L.scale_fields('skeleton250')
    oc.ref_configure()
    ra, ri, rt = oc.ref_decode(f['cif'], stride, f['caf'], stride, f['skeleton'], 133, taps=True)
    oa, oi, ot = oc.decode(f['cif'], stride, f['caf'], stride, f['skeleton'], 133, taps=True)
    np.testing.assert_array_equal(rt['cifhr'], ot['cifhr'])
    for a, b in zip(rt['fwd'] + rt['bwd'], ot['fwd'] + ot['bwd']):
        np.testing.assert_array_equal(a, b)
    np.testing.assert_array_equal(ra, oa)
    np.testing.assert_array_equal(ri, oi)


# ---- 3. one batch mixing a crowd, a single person, an empty image and a small group

def test_mixed_batch_equals_single_decodes_and_oracle():
    names = ['coco60_81x81_s8', 'coco1_81x81_s8', 'coco0_81x81_s8', 'coco10_81x81_s8']
    fs = [L.scale_fields(n)[0] for n in names]
    d = decoder.CifCaf(17, torch.from_numpy(fs[0]['skeleton']))
    cif = torch.from_numpy(np.stack([f['cif'] for f in fs])).cuda()
    caf = torch.from_numpy(np.stack([f['caf'] for f in fs])).cuda()
    res = d.decode_batch(cif, 8, caf, 8)
    single = decoder.CifCaf(17, torch.from_numpy(fs[0]['skeleton']))
    for b, (name, f) in enumerate(zip(names, fs)):
        oa, oi, ot = oracle(f, 8)
        assert_stages_equal(d, ot, image=b)
        sa, si = single.call(torch.from_numpy(f['cif']), 8, torch.from_numpy(f['caf']), 8)
        assert torch.equal(res[b][0], sa) and torch.equal(res[b][1], si), name
        helpers.assert_annotations_close(sa.numpy(), oa, name)
        np.testing.assert_array_equal(si.numpy(), oi)
    assert [len(r[0]) for r in res][1:3] == [1, 0]


# ---- 4. the deferral radius of k_grow changes the schedule, never the result

@pytest.mark.parametrize('names', [['coco60_81x81_s8', 'coco10_81x81_s8', 'ties_saturated'], ['skeleton800']],
                         ids=['coco_crowd', 'one_worker'])
def test_grow_deferral_never_changes_the_result(monkeypatch, names):
    fs = [L.scale_fields(n) for n in names]
    stride = fs[0][1]
    sk = torch.from_numpy(fs[0][0]['skeleton'])
    K = fs[0][0]['n_keypoints']
    cif = torch.from_numpy(np.stack([f['cif'] for f, _, _ in fs])).cuda()
    caf = torch.from_numpy(np.stack([f['caf'] for f, _, _ in fs])).cuda()
    want = [oracle(f, stride)[:2] for f, _, _ in fs]
    results, schedules = [], []
    for radius in ('0', '0.5', '6', '1e6'):
        monkeypatch.setenv('PIFPAF_GROW_DEFER', radius)      # read when the native handle is created
        d = decoder.CifCaf(K, sk)
        res = d.decode_batch(cif, stride, caf, stride)
        st = d.last_stats()
        schedules.append((st['grow_rounds'], st['grow_seeds_grown']))
        results.append(res)
        for (ga, gi), (oa, oi), name in zip(res, want, names):
            helpers.assert_annotations_close(ga.numpy(), oa, f'{name} defer {radius}')
            np.testing.assert_array_equal(gi.numpy(), oi)
    for res in results[1:]:
        for (a0, i0), (a1, i1) in zip(results[0], res):
            assert torch.equal(a0, a1) and torch.equal(i0, i1)
    if L.plan_grow(K, sk.shape[0])[0] > 1:
        assert len(set(schedules)) > 1, schedules


# ---- 5. exact ties between seed scores, across 1024-seed sort tiles and across fields

@pytest.mark.parametrize('name', ['ties_saturated', 'ties_levels', 'ties_uniform'])
def test_seed_ties_keep_fill_order(name):
    _, ot, _ = single_decode(name)
    v = ot['seeds_vxys'][:, 0]
    vals, counts = np.unique(v, return_counts=True)
    top = vals[np.argmax(counts)]
    assert counts.max() > 4 * 1024 and len(set(ot['seeds_f'][v == top].tolist())) > 8
    if name == 'ties_uniform':
        assert len(vals) == 1       # every candidate scores 1.0: all four radix passes are skipped


def det_tie_field(n_objects, seed):
    f = synth.make_det_fields(91, 81, 81, n_objects, seed, n_distractors=20)['field']
    f[:, 1] = L.tie_quantise(f[:, 1], 'saturate')
    return f


def test_cifdet_seed_ties_keep_fill_order():
    fields = [det_tie_field(n, 600 + n) for n in (150, 400)]
    p = oc.default_params(seed_sort_stable=1)
    d = decoder.CifDet()
    try:
        decoder.CifDet.set_max_detections_before_nms(1000)
        got = d.decode_batch(torch.from_numpy(np.stack(fields)).cuda(), 8)
        for f, (gc, gs, gb) in zip(fields, got):
            wc, ws, wb, t = oc.decode_det(f, 8, params=p, max_detections_before_nms=1000, taps=True)
            v = t['seeds_vxywh'][:, 0]
            assert (v == 1.0).sum() > 1024 and len(set(t['seeds_f'][v == 1.0].tolist())) > 8
            assert (ws == 1.0).sum() > 100
            np.testing.assert_array_equal(gc.numpy(), wc)
            np.testing.assert_array_equal(gs.numpy(), ws)
            np.testing.assert_array_equal(gb.numpy(), wb)
    finally:
        decoder.CifDet.set_max_detections_before_nms(120)


# ---- 6. max_annotations at its exact boundary

@pytest.mark.parametrize('with_initial', [False, True])
def test_annotation_capacity_boundary(with_initial):
    f, stride, _ = L.scale_fields('coco60_81x81_s8')
    init = ids = None
    if with_initial:
        base, _ = oc.decode(f['cif'], stride, f['caf'], stride, f['skeleton'], 17,
                            params=oc.default_params(seed_sort_stable=1))
        init = base[:5].copy()
        init[:, 9:] = 0.0
        ids = np.arange(100, 105, dtype=np.int64)
    p = oc.default_params(seed_sort_stable=1)
    oa, oi, ot = oc.decode(f['cif'], stride, f['caf'], stride, f['skeleton'], 17, params=p, taps=True,
                           initial_annotations=init, initial_ids=ids)
    n = ot['n_pre_nms']
    assert n > len(oa) > 50

    def run(cap):
        d = decoder.CifCaf(17, torch.from_numpy(f['skeleton']))
        d.max_annotations = cap
        args = (torch.from_numpy(f['cif']), stride, torch.from_numpy(f['caf']), stride)
        if with_initial:
            return d.call_with_initial_annotations(*args, torch.from_numpy(init), torch.from_numpy(ids))
        return d.call(*args)

    ga, gi = run(n)
    helpers.assert_annotations_close(ga.numpy(), oa, f'max_annotations {n}')
    np.testing.assert_array_equal(gi.numpy(), oi)
    with pytest.raises(RuntimeError, match='capacity'):
        run(n - 1)


# ---- 7. packed results larger than the 512 KB fetch prefix

PREFIX = 512 * 1024
FETCH_POOLS = {     # images of one shape with many, some, one and no annotations
    'coco': ['coco60_81x81_s8', 'coco10_81x81_s8', 'coco1_81x81_s8', 'coco0_81x81_s8'],
    'wholebody': ['wholebody8_41x41', 'wholebody1_41x41', 'wholebody0_41x41'],
}


def header_bytes(B):
    return ((3 * B + 1) * 4 + 15) & ~15


def needs_tail(total, B, max_batch, K):
    """does a batch of B images with `total` annotations on a handle reserved for max_batch need the second copy"""
    return header_bytes(B) + total * (K + 1) * 16 > header_bytes(max_batch) + PREFIX


def compose(counts, B, target):
    """B image indices (greedy, largest count first) whose annotation counts sum to target"""
    order, left = [], target
    for i in sorted(range(len(counts)), key=lambda i: -counts[i]):
        while counts[i] > 0 and left >= counts[i] and len(order) < B:
            order.append(i)
            left -= counts[i]
    order += [counts.index(0)] * (B - len(order))
    assert left == 0 and len(order) == B, (counts, B, target)
    return order


class FetchPool:
    """the images of FETCH_POOLS[pool], their single decodes (checked against the oracle) and batches of them"""
    def __init__(self, pool):
        self.fields = [L.scale_fields(n)[0] for n in FETCH_POOLS[pool]]
        self.stride = L.scale_fields(FETCH_POOLS[pool][0])[1]
        self.K = self.fields[0]['n_keypoints']
        self.skeleton = torch.from_numpy(self.fields[0]['skeleton'])
        single = decoder.CifCaf(self.K, self.skeleton)
        self.want = []
        for f in self.fields:
            ga, gi = single.call(torch.from_numpy(f['cif']), self.stride, torch.from_numpy(f['caf']), self.stride)
            oa, oi, _ = oracle(f, self.stride)
            helpers.assert_annotations_close(ga.numpy(), oa, 'single decode')
            np.testing.assert_array_equal(gi.numpy(), oi)
            self.want.append((ga, gi))
        self.counts = [len(a) for a, _ in self.want]

    def order(self, B, max_batch, tail):
        """a batch on the last annotation count that fits the prefix (tail=False) or the first that does not"""
        limit = max(t for t in range(B * max(self.counts) + 1) if not needs_tail(t, B, max_batch, self.K))
        return compose(self.counts, B, limit + 1 if tail else limit)

    def batch(self, order):
        cif = torch.from_numpy(np.stack([self.fields[i]['cif'] for i in order])).cuda()
        caf = torch.from_numpy(np.stack([self.fields[i]['caf'] for i in order])).cuda()
        return cif, caf

    def decoder(self, max_batch):
        """a fresh handle: its pinned result buffers hold no records of an earlier fetch"""
        d = decoder.CifCaf(self.K, self.skeleton)
        d.reserve(max_batch, *self.fields[0]['cif'].shape[2:], self.stride)
        return d

    def check(self, res, order):
        assert len(res) == len(order)
        for b, (i, (ga, gi)) in enumerate(zip(order, res)):
            assert torch.equal(ga, self.want[i][0]) and torch.equal(gi, self.want[i][1]), f'image {b}'


@pytest.mark.parametrize('pool,B,max_batch', [('coco', 48, 48), ('coco', 40, 64), ('wholebody', 40, 40)],
                         ids=['coco', 'coco_batch_below_reserved', 'wholebody'])
def test_fetch_beyond_the_prefix(pool, B, max_batch):
    fp = FetchPool(pool)
    for tail in (True, False):
        order = fp.order(B, max_batch, tail)
        total = sum(fp.counts[i] for i in order)
        assert needs_tail(total, B, max_batch, fp.K) == tail
        d = fp.decoder(max_batch)
        cif, caf = fp.batch(order)
        res = d.decode_batch(cif, fp.stride, caf, fp.stride)
        assert sum(len(r[0]) for r in res) == total
        fp.check(res, order)


@pytest.mark.parametrize('older_needs_tail', [True, False])
def test_fetch_beyond_the_prefix_pipelined(older_needs_tail):
    """two fetches outstanding on one handle; only one of them needs the tail copy"""
    B = 48
    fp = FetchPool('coco')
    orders = [fp.order(B, B, True), fp.order(B, B, False)]
    orders[1] = orders[1][::-1]          # other images in the places of the first batch's tail records
    if not older_needs_tail:
        orders = orders[::-1]
    d = fp.decoder(B)
    keep = []
    for order in orders:
        cif, caf = fp.batch(order)
        keep.append((cif, caf))
        d.decode_batch_async(cif, fp.stride, caf, fp.stride)
        d.fetch_begin()
    for order in orders:
        fp.check(d.fetch_end(), order)


# ---- 8. CifDet at the handle's capacity

@pytest.mark.parametrize('cap,n_objects', [(1000, 1400), (4096, 5200)])
def test_cifdet_at_capacity(cap, n_objects):
    torchvision = pytest.importorskip('torchvision')
    field = synth.make_det_fields(91, 81, 81, n_objects, 700 + cap, n_distractors=40, n_overlapping=60)['field']
    want = oc.decode_det(field, 8, params=oc.default_params(seed_sort_stable=1), max_detections_before_nms=cap)
    assert len(want[0]) == cap                  # more raw detections than the limit
    d = decoder.CifDet()
    if cap > d.max_detections:
        d.max_detections = cap
    dev = torch.from_numpy(field[None]).cuda()
    try:
        decoder.CifDet.set_max_detections_before_nms(cap)
        (cats, scores, boxes), = d.decode_batch(dev, 8)
        for g, w in zip((cats, scores, boxes), want):
            np.testing.assert_array_equal(g.numpy(), w)
        for by_category in (True, False):
            (gc, gs, gb), = d.decode_batch(dev, 8, nms=True, iou_threshold=0.5, nms_by_category=by_category,
                                           suppression=0.1, instance_threshold=0.15)
            if by_category:
                keep = torchvision.ops.batched_nms(boxes, scores, cats, 0.5)
            else:
                keep = torchvision.ops.nms(boxes, scores, 0.5)
            s = scores.clone() * 0.1
            s[keep] = scores[keep]
            mask = s > 0.15
            assert 0 < int(mask.sum()) < cap
            assert torch.equal(gc, cats[mask]) and torch.equal(gs, s[mask]) and torch.equal(gb, boxes[mask])
    finally:
        decoder.CifDet.set_max_detections_before_nms(120)


# ---- handles with different shared-memory plans in one process

def test_handles_with_different_shared_memory_plans_coexist():
    """The dynamic shared-memory limit of a kernel belongs to the device, not to a handle: creating a handle whose
    plan needs less (a 1-worker grow CTA; a CifDet NMS for 1024 detections) must not break the launches of an older
    handle that needs more."""
    f, stride, _ = L.scale_fields('coco10_81x81_s8')
    fw, _, _ = L.scale_fields('skeleton800')
    assert L.plan_grow(17, 19)[3] > L.plan_grow(133, fw['skeleton'].shape[0])[3]
    args = (torch.from_numpy(f['cif']), stride, torch.from_numpy(f['caf']), stride)
    wide = (torch.from_numpy(fw['cif']), stride, torch.from_numpy(fw['caf']), stride)
    coco = decoder.CifCaf(17, torch.from_numpy(f['skeleton']))
    first = coco.call(*args)
    decoder.CifCaf(133, torch.from_numpy(fw['skeleton'])).call(*wide)
    again = coco.call(*args)
    assert torch.equal(first[0], again[0]) and torch.equal(first[1], again[1])

    field = torch.from_numpy(synth.make_det_fields(91, 41, 41, 300, 31, n_overlapping=20)['field'][None]).cuda()
    big = decoder.CifDet()
    big.max_detections = 4096
    try:
        decoder.CifDet.set_max_detections_before_nms(4096)
        first = big.decode_batch(field, 8, nms=True)[0]
        decoder.CifDet.set_max_detections_before_nms(120)
        decoder.CifDet().decode_batch(field, 8, nms=True)
        decoder.CifDet.set_max_detections_before_nms(4096)
        again = big.decode_batch(field, 8, nms=True)[0]
    finally:
        decoder.CifDet.set_max_detections_before_nms(120)
    for a, b in zip(first, again):
        assert torch.equal(a, b)
