"""GPU: the pose (CifCaf) and CifDet handles share one front end in decoder.cu -- CifHr, seeds, the occupancy map and
their workspace.  Pinned here: the kernels each decode launches, that a create refused for lack of memory leaves
every other handle of the thread working, and that two handles used in turn on one stream keep their own state."""
import ctypes

import numpy as np
import pytest
import torch

import helpers
from openpifpaf_b200 import _lib, constants, decoder, synth
from oracle import cifcaf as oc

pytestmark = pytest.mark.gpu


def launches(fn):
    """library kernel launches made by fn()"""
    L = _lib.lib()
    n0 = L.pifpaf_launch_count()
    fn()
    torch.cuda.synchronize()
    return int(L.pifpaf_launch_count() - n0)


def pose_case(seed):
    f = synth.make_fields('cocokp', 17, 21, 2, seed, n_distractors=4)
    d = decoder.CifCaf(17, torch.from_numpy(f['skeleton']))
    cif = torch.from_numpy(f['cif'][None]).cuda()
    caf = torch.from_numpy(f['caf'][None]).cuda()
    want, _ = oc.decode(f['cif'], 16, f['caf'], 16, f['skeleton'], 17, params=oc.default_params(seed_sort_stable=1))
    return d, cif, caf, want


def det_case(seed):
    fields = [synth.make_det_fields(80, 23, 37, n, seed + n, n_distractors=5)['field'] for n in (3, 40)]
    want = [oc.decode_det(f, 8, params=oc.default_params(seed_sort_stable=1)) for f in fields]
    return decoder.CifDet(), torch.from_numpy(np.stack(fields)).cuda(), want


def assert_det_equal(got, want):
    for (gc, gs, gb), (wc, ws, wb) in zip(got, want):
        np.testing.assert_array_equal(gc.numpy(), wc)
        np.testing.assert_array_equal(gs.numpy(), ws)
        np.testing.assert_array_equal(gb.numpy(), wb)


@pytest.mark.parametrize('static, want', [(None, 8), (('CifCaf', 'force_complete'), 10),
                                          (('CifHr', 'ablation_skip'), 6)],
                         ids=['default', 'force_complete', 'cifhr_ablation_skip'])
def test_pose_decode_launch_sequence(static, want):
    """compact, tiles, candidates, sort, caf_scored, grow, nms, pack; force_complete adds caf_scored and
    force_complete; the CifHr ablation drops compact and tiles"""
    d, cif, caf, _ = pose_case(941)
    setter = getattr(getattr(decoder, static[0]), 'set_' + static[1]) if static else None
    if setter:
        setter(True)
    try:
        d.decode_batch(cif, 16, caf, 16)          # creates the handle
        n = launches(lambda: d.decode_batch(cif, 16, caf, 16))
    finally:
        if setter:
            setter(False)
    print('pose', static, 'launches', n)
    assert n == want


@pytest.mark.parametrize('nms, want', [(False, 5), (True, 6)])
def test_cifdet_decode_launch_sequence(nms, want):
    """compact, tiles, candidates, sort, select; nms adds k_det_nms"""
    d, field, _ = det_case(950)
    d.decode_batch(field, 8, nms=nms)
    n = launches(lambda: d.decode_batch(field, 8, nms=nms))
    print('cifdet nms', nms, 'launches', n)
    assert n == want


@pytest.mark.parametrize('failing', ['pose', 'cifdet'])
def test_failed_create_leaves_library_usable(failing):
    """A create whose CifHr map alone needs more than a terabyte is refused with E_NOMEM.  The runtime error of that
    cudaMalloc must not surface as a launch failure of the next decode on another handle of the thread."""
    L = _lib.lib()
    handle = ctypes.c_void_p()
    if failing == 'pose':
        sk = np.asarray(constants.COCO_PERSON_SKELETON, dtype=np.int64) - 1
        rc = L.pifpaf_decoder_create(ctypes.byref(handle), 0, 17, 17, sk.shape[0], sk.ctypes.data_as(ctypes.c_void_p),
                                     4, 8192, 8192, 8, 512)          # CifHr: 4 x 17 x 65529 x 65536 f32, ~1.2 TB
    else:
        rc = L.pifpaf_cifdet_create(ctypes.byref(handle), 0, 91, 1, 8192, 8192, 8, 1024)   # CifHr ~1.6 TB
    assert rc == _lib.E_NOMEM, (rc, L.pifpaf_last_error())
    assert not handle.value
    d, cif, caf, want = pose_case(961)
    helpers.assert_annotations_close(d.decode_batch(cif, 16, caf, 16)[0][0].numpy(), want, 'pose')
    d, field, want = det_case(970)
    assert_det_equal(d.decode_batch(field, 8), want)


def test_interleaved_pose_and_cifdet_handles_keep_their_own_state():
    """300 rounds of pose then CifDet on one stream: the occupancy tags of both wrap (pose every 127 decodes, CifDet
    after 254), and the last round still equals the first and the oracle"""
    pose, cif, caf, want_pose = pose_case(981)
    det, field, want_det = det_case(990)
    st = torch.cuda.current_stream()
    first = None
    for i in range(300):
        rp = pose.decode_batch(cif, 16, caf, 16, stream=st)
        rd = det.decode_batch(field, 8, stream=st)
        if i == 0:
            first = rp
        if i in (0, 299):
            helpers.assert_annotations_close(rp[0][0].numpy(), want_pose, f'pose, round {i}')
            assert torch.equal(rp[0][0], first[0][0]) and torch.equal(rp[0][1], first[0][1]), i
            assert_det_equal(rd, want_det)
    assert len(want_pose) == 2 and min(len(w[0]) for w in want_det) >= 3
