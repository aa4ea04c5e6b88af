"""GPU: the CUDA decoders under every decoder option of the reference (oracle/make_golden.py OPTION_CASES) and at
CifHr revisions other than 1.0, against the plain-C oracle: CifHr map, seeds and CAF lists bit for bit, annotations
within the parity tolerances, ids equal.  CifDet's NMS is checked against torchvision on CPU tensors, as the reference's
wrapper runs it (decoder/cifdet.py:60-68), including above 1000 detections, where torchvision's batched_nms switches
from the coordinate trick to one nms per category."""
import numpy as np
import pytest
import torch

import decoder_layout as L
import helpers
from openpifpaf_b200 import decoder, synth
from oracle import cifcaf as oc, make_golden

pytestmark = pytest.mark.gpu

OPTIONS = dict([('default', {})] + make_golden.OPTION_CASES)
REVISIONS = (0, 2, 4097, 10000)
_CASES = {name: args for name, *args in make_golden.CASES}
FIELDS = make_golden.OPTION_FIELDS + ['coco60_81x81_s8', 'wholebody8_41x41']

# reference static (make_golden / ref_configure name) -> native static
NATIVE = {
    'block_joints': (decoder.CifCaf, 'block_joints'), 'greedy': (decoder.CifCaf, 'greedy'),
    'keypoint_threshold': (decoder.CifCaf, 'keypoint_threshold'),
    'keypoint_threshold_rel': (decoder.CifCaf, 'keypoint_threshold_rel'),
    'reverse_match': (decoder.CifCaf, 'reverse_match'), 'force_complete': (decoder.CifCaf, 'force_complete'),
    'force_complete_caf_th': (decoder.CifCaf, 'force_complete_caf_th'),
    'cifhr_neighbors': (decoder.CifHr, 'neighbors'), 'cifhr_threshold': (decoder.CifHr, 'threshold'),
    'cifhr_ablation_skip': (decoder.CifHr, 'ablation_skip'),
    'seed_threshold': (decoder.CifSeeds, 'threshold'), 'seeds_ablation_nms': (decoder.CifSeeds, 'ablation_nms'),
    'seeds_ablation_no_rescore': (decoder.CifSeeds, 'ablation_no_rescore'),
    'caf_score_th': (decoder.CafScored, 'default_score_th'),
    'caf_ablation_no_rescore': (decoder.CafScored, 'ablation_no_rescore'),
    'nms_instance_threshold': (decoder.NMSKeypoints, 'instance_threshold'),
    'nms_keypoint_threshold': (decoder.NMSKeypoints, 'keypoint_threshold'),
    'nms_suppression': (decoder.NMSKeypoints, 'suppression'),
}


@pytest.fixture(autouse=True)
def restore_statics():
    """files that run later assume the default statics"""
    yield
    helpers.reset_native_statics()


def configure(statics):
    helpers.reset_native_statics()
    for k, v in statics.items():
        cls, name = NATIVE[k]
        getattr(cls, 'set_' + name)(v)


def fields(name):
    if name in _CASES:
        workload, h, w, n_people, seed, n_dis, stride, _ = _CASES[name]
        return synth.make_fields(workload, h, w, n_people, seed, n_dis), stride
    f, stride, _ = L.scale_fields(name)
    return f, stride


def oracle(f, stride, statics, revision=1.0):
    p = oc.default_params(seed_sort_stable=1, cifhr_revision=float(revision), **helpers.statics_to_params(statics))
    return oc.decode(f['cif'], stride, f['caf'], stride, f['skeleton'], f['n_keypoints'], params=p, taps=True)


def check(d, got, want, statics, what):
    (ga, gi), (oa, oi, ot) = got, want
    np.testing.assert_array_equal(d.tap_cifhr().numpy(), ot['cifhr'], err_msg=what)
    sf, sv = d.tap_seeds()
    np.testing.assert_array_equal(sf.numpy(), ot['seeds_f'], err_msg=what)
    np.testing.assert_array_equal(sv.numpy(), ot['seeds_vxys'], err_msg=what)
    if not statics.get('force_complete'):
        fw, bw = d.tap_caf()
        for c, (a, b) in enumerate(zip(fw + bw, ot['fwd'] + ot['bwd'])):
            np.testing.assert_array_equal(a.numpy(), b, err_msg=f'{what}: CAF list {c}')
    helpers.assert_annotations_close(ga.numpy(), oa, what)
    np.testing.assert_array_equal(gi.numpy(), oi, err_msg=what)


def make_decoder(f):
    """kp_rel_1 and neighbors_64 keep hundreds of annotations before NMS on the crowd inputs"""
    d = decoder.CifCaf(f['n_keypoints'], torch.from_numpy(f['skeleton']))
    d.max_annotations = 4096
    return d


def decode(d, f, stride):
    return d.call(torch.from_numpy(f['cif']), stride, torch.from_numpy(f['caf']), stride)


@pytest.mark.parametrize('field', FIELDS)
@pytest.mark.parametrize('option', list(OPTIONS))
def test_cuda_matches_oracle_under_option(option, field):
    """(neighbors 1 saturates the map into exact seed ties: the oracle sorts stably, like the kernels; that the
    reference's introsort order agrees with the oracle's is test_decoder_options.py's part)"""
    statics = OPTIONS[option]
    f, stride = fields(field)
    configure(statics)
    d = make_decoder(f)
    check(d, decode(d, f, stride), oracle(f, stride, statics), statics, f'{option} {field}')


@pytest.mark.parametrize('option', ['default', 'cif_th_0.05', 'neighbors_1', 'seeds_nms', 'no_rescore_skip',
                                    'caf_no_rescore', 'force_complete', 'eval'])
def test_cuda_matches_oracle_at_revisions(monkeypatch, option):
    statics = OPTIONS[option]
    configure(statics)
    params = decoder.CifCaf.params
    for field in ('coco41_poisson_s0', 'wholebody_4p'):
        f, stride = fields(field)
        for r in REVISIONS:
            monkeypatch.setattr(decoder.CifCaf, 'params',
                                classmethod(lambda cls, _r=r, **kw: params(**{'cifhr_revision': float(_r), **kw})))
            d = make_decoder(f)
            got = decode(d, f, stride)
            assert d.get_cifhr()[1] == float(r)
            check(d, got, oracle(f, stride, statics, r), statics, f'{option} {field} revision {r}')


def test_one_handle_decodes_every_option_in_sequence():
    """occupancy and CifHr epoch tags, force-complete list refills and the ablation_skip tap carry nothing from one
    option set to the next: one handle equals a fresh handle per option set"""
    f, stride = fields('crowd30')
    shared = make_decoder(f)
    for option, statics in list(OPTIONS.items()) * 2:
        configure(statics)
        fresh = make_decoder(f)
        want = decode(fresh, f, stride)
        got = decode(shared, f, stride)
        assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1]), option
        assert torch.equal(shared.tap_cifhr(), fresh.tap_cifhr()), option
        assert all(torch.equal(a, b) for a, b in zip(shared.tap_seeds(), fresh.tap_seeds())), option


# ---- CifDet

def det_oracle(field, stride, revision=1.0, max_det=120, **params):
    p = oc.default_params(seed_sort_stable=1, cifhr_revision=float(revision), **params)
    return oc.decode_det(field, stride, params=p, max_detections_before_nms=max_det)


def assert_det_equal(got, want, what):
    for g, w in zip(got, want):
        np.testing.assert_array_equal(g.numpy(), w, err_msg=what)


@pytest.mark.parametrize('statics', [{}, {'cifhr_threshold': 0.1}, {'cifhr_threshold': 0.5}, {'cifhr_neighbors': 1},
                                     {'cifhr_neighbors': 64}, {'seed_threshold': 0.05}, {'seed_threshold': 0.5}],
                         ids=['default', 'cif_th_0.1', 'cif_th_0.5', 'neighbors_1', 'neighbors_64', 'seed_th_0.05',
                              'seed_th_0.5'])
def test_cifdet_matches_oracle_under_options_and_revisions(monkeypatch, statics):
    field = synth.make_det_fields(80, 41, 41, 60, 17, n_distractors=12, n_overlapping=6)['field']
    decoder.CifHr.set_neighbors(statics.get('cifhr_neighbors', 16))
    decoder.CifHr.set_threshold(statics.get('cifhr_threshold', 0.3))
    decoder.CifDetSeeds.set_threshold(statics.get('seed_threshold', 0.2))
    params = decoder.CifDet.params
    for r in (1,) + REVISIONS:
        monkeypatch.setattr(decoder.CifDet, 'params',
                            classmethod(lambda cls, _r=r, **kw: params(**{'cifhr_revision': float(_r), **kw})))
        d = decoder.CifDet()
        want = det_oracle(field, 16, r, **statics)
        assert len(want[0]) > 0
        assert_det_equal(d.call(torch.from_numpy(field), 16), want, f'{statics} revision {r}')


def nms_like_reference(cats, scores, boxes, iou_threshold, nms_by_category, suppression, instance_threshold):
    """decoder/cifdet.py:60-71 on CPU tensors: torchvision's NMS, the suppression of what it drops, the score filter"""
    import torchvision
    if nms_by_category:
        keep = torchvision.ops.batched_nms(boxes, scores, cats, iou_threshold)
    else:
        keep = torchvision.ops.nms(boxes, scores, iou_threshold)
    s = scores.clone() * suppression
    s[keep] = scores[keep]
    mask = s > instance_threshold
    return cats[mask], s[mask], boxes[mask]


def assert_nms_equal(d, dev, stride, raw, **nms):
    (gc, gs, gb), = d.decode_batch(dev, stride, nms=True, **nms)
    wc, ws, wb = nms_like_reference(*raw, **nms)
    assert torch.equal(gc, wc) and torch.equal(gs, ws) and torch.equal(gb, wb), nms
    return len(wc)


@pytest.mark.parametrize('iou_threshold', [0.0, 0.3, 0.5, 1.0])
def test_cifdet_nms_options_equal_torchvision(iou_threshold):
    pytest.importorskip('torchvision')
    field = synth.make_det_fields(6, 41, 41, 80, 900, n_distractors=10, n_overlapping=20)['field']
    d = decoder.CifDet()
    dev = torch.from_numpy(field[None]).cuda()
    (cats, scores, boxes), = d.decode_batch(dev, 16)
    assert len(cats) > 100
    raw = (cats, scores, boxes)
    top = float(scores.max())
    for by_category in (True, False):
        for suppression in (0.0, 1.0, 0.1):
            for instance_threshold in (0.0, top):
                n = assert_nms_equal(d, dev, 16, raw, iou_threshold=iou_threshold, nms_by_category=by_category,
                                     suppression=suppression, instance_threshold=instance_threshold)
                if instance_threshold == top:
                    assert n == 0
                elif suppression > 0.0 or iou_threshold == 1.0:
                    assert n == len(cats)


# ---- more than 1000 raw detections: torchvision's per-category batched_nms

def crafted_det_field(seed, n_filler):
    """a CifDet field [91,6,81,81] whose every box is one cell's vote (stride 8, CifHr.neighbors = 1 so that a lone cell
    seeds at its own confidence):
    - 40 category pairs: a box around the top-left corner (negative x1, y1; cifdet.cpp:62 does not clip) in category c
      and a bottom-right box at the largest coordinate of the image in c - 1.  Shifted by c * (max + 1), the first
      overlaps the second at IoU ~0.12;
    - 300 pairs in categories 60-90 of two 100-pixel boxes 100/3 pixels apart (IoU 0.5 +- 1e-4): far enough apart that
      the occupancy map keeps both seeds, close enough to threshold that shifted coordinates round across it;
    - small boxes in categories 0-59 up to more than 1000 detections."""
    rng = np.random.Generator(np.random.PCG64(seed))
    F, h, w, stride = 91, 81, 81, 8
    field = np.zeros((F, 6, h, w), dtype=np.float32)
    used = np.zeros((F,), dtype=np.int64)

    def box(f, cx, cy, bw, bh, conf):
        k = int(used[f])
        used[f] += 1
        j, i = divmod(k, w)
        field[f, :, j, i] = (0.0, conf, cx / stride, cy / stride, bw / stride, bh / stride)

    for c in range(1, 41):
        box(c, 2.0, 2.0, 96.0, 96.0, 0.5 + 0.4 * rng.random())
        box(c - 1, 636.0, 636.0, 96.0, 96.0, 0.5 + 0.4 * rng.random())
    for k in range(300):
        f = 60 + k % 31
        cx, cy = 120.0 + 40.0 * (k // 31), 100.0 + 150.0 * (k % 3)
        d = 100.0 / 3.0 + 0.01 * (rng.random() - 0.5) * 2
        box(f, cx, cy, 100.0, 100.0, 0.5 + 0.4 * rng.random())
        box(f, cx + d, cy, 100.0, 100.0, 0.5 + 0.4 * rng.random())
    for k in range(n_filler):
        f = k % 60
        cx, cy = 60.0 + 16.0 * ((k // 60) % 32), 60.0 + 16.0 * (k // (60 * 32)) + 24.0 * (f % 20)
        box(f, cx, cy, 6.0 + 4.0 * rng.random(), 6.0 + 4.0 * rng.random(), 0.3 + 0.6 * rng.random())
    return field, stride


@pytest.mark.parametrize('cap,n_filler', [(1500, 650), (2048, 1200)])
def test_cifdet_nms_above_1000_detections_is_per_category(cap, n_filler):
    torchvision = pytest.importorskip('torchvision')
    from torchvision.ops import boxes as tvb
    field, stride = crafted_det_field(cap, n_filler)
    decoder.CifHr.set_neighbors(1)
    decoder.CifDet.set_max_detections_before_nms(cap)
    want = det_oracle(field, stride, max_det=cap, cifhr_neighbors=1)
    n = len(want[0])
    assert 1000 < n < cap
    d = decoder.CifDet()
    d.max_detections = cap
    dev = torch.from_numpy(field[None]).cuda()
    (cats, scores, boxes), = d.decode_batch(dev, stride)
    assert_det_equal((cats, scores, boxes), want, 'raw detections')
    # the oracle (cifdet.cpp) keeps the negative-corner boxes and both boxes of every near-threshold pair
    assert int(((boxes[:, 0] < 0) & (boxes[:, 1] < 0)).sum()) == 40
    assert int((cats >= 61).sum()) == 600
    for iou in (0.1, 0.5):
        trick = tvb._batched_nms_coordinate_trick(boxes, scores, cats, iou)
        vanilla = tvb._batched_nms_vanilla(boxes, scores, cats, iou)
        assert set(trick.tolist()) != set(vanilla.tolist()), iou       # the input tells the two apart
        assert torch.equal(torchvision.ops.batched_nms(boxes, scores, cats, iou), vanilla)
        for suppression in (0.0, 0.1):
            assert_nms_equal(d, dev, stride, (cats, scores, boxes), iou_threshold=iou, nms_by_category=True,
                             suppression=suppression, instance_threshold=0.0)
        assert_nms_equal(d, dev, stride, (cats, scores, boxes), iou_threshold=iou, nms_by_category=False,
                         suppression=0.1, instance_threshold=0.15)


def test_cifdet_nms_at_1000_detections_keeps_the_coordinate_trick():
    """the last count torchvision runs with the coordinate trick"""
    pytest.importorskip('torchvision')
    field, stride = crafted_det_field(1500, 650)
    decoder.CifHr.set_neighbors(1)
    decoder.CifDet.set_max_detections_before_nms(1000)
    d = decoder.CifDet()
    dev = torch.from_numpy(field[None]).cuda()
    (cats, scores, boxes), = d.decode_batch(dev, stride)
    assert len(cats) == 1000
    assert_nms_equal(d, dev, stride, (cats, scores, boxes), iou_threshold=0.1, nms_by_category=True,
                     suppression=0.1, instance_threshold=0.0)
