"""ctypes wrapper of the plain-C oracle (oracle/cifcaf_oracle.c) and loader of the
compiled unmodified reference (oracle/_ref/refcpp.so).  TEST INFRASTRUCTURE ONLY."""
import ctypes
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, '_build', 'libcifcaf_oracle.so')
REF_SO = os.path.join(HERE, '_ref', 'refcpp.so')


class OracleParams(ctypes.Structure):
    """Mirror of oracle_params_t."""
    _fields_ = [
        ('cifhr_neighbors', ctypes.c_int64),
        ('cifhr_threshold', ctypes.c_double),
        ('cifhr_ablation_skip', ctypes.c_int32),
        ('seed_threshold', ctypes.c_double),
        ('seeds_ablation_nms', ctypes.c_int32),
        ('seeds_ablation_no_rescore', ctypes.c_int32),
        ('caf_score_th', ctypes.c_double),
        ('caf_cif_floor', ctypes.c_double),
        ('caf_ablation_no_rescore', ctypes.c_int32),
        ('block_joints', ctypes.c_int32),
        ('greedy', ctypes.c_int32),
        ('keypoint_threshold', ctypes.c_double),
        ('keypoint_threshold_rel', ctypes.c_double),
        ('reverse_match', ctypes.c_int32),
        ('force_complete', ctypes.c_int32),
        ('force_complete_caf_th', ctypes.c_double),
        ('nms_suppression', ctypes.c_double),
        ('nms_instance_threshold', ctypes.c_double),
        ('nms_keypoint_threshold', ctypes.c_double),
        ('occ_reduction', ctypes.c_double),
        ('occ_min_scale', ctypes.c_double),
        ('cifhr_revision', ctypes.c_double),
        ('seed_sort_stable', ctypes.c_int32),
    ]


_lib = None


def build():
    subprocess.check_call(['make', '-s', '-C', HERE])
    return LIB_PATH


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH) or \
                os.path.getmtime(LIB_PATH) < os.path.getmtime(os.path.join(HERE, 'cifcaf_oracle.c')):
            build()
        _lib = ctypes.CDLL(LIB_PATH)
        _lib.oracle_cifcaf_call.restype = ctypes.c_int64
        _lib.oracle_cifseeds.restype = ctypes.c_int64
        _lib.oracle_cifdet_call.restype = ctypes.c_int64
    return _lib


def default_params(**overrides):
    p = OracleParams()
    lib().oracle_default_params(ctypes.byref(p))
    for k, v in overrides.items():
        assert hasattr(p, k), k
        setattr(p, k, v)
    return p


def _ptr(a, ctype):
    return a.ctypes.data_as(ctypes.POINTER(ctype)) if a is not None else None


def decode(cif, cif_stride, caf, caf_stride, skeleton, n_keypoints=None, params=None,
           initial_annotations=None, initial_ids=None, taps=False, cap=None):
    """Oracle equivalent of CifCaf(n_keypoints, skeleton).call_with_initial_annotations(...)
    on a FRESH instance.  cif [F,5,h,w], caf [C,8,h,w] float32 numpy; skeleton [C,2] 0-based.
    Returns (annotations [N,K,4] f32, ids [N] i64[, taps dict])."""
    cif = np.ascontiguousarray(cif, dtype=np.float32)
    caf = np.ascontiguousarray(caf, dtype=np.float32)
    skeleton = np.ascontiguousarray(skeleton, dtype=np.int64)
    F, _, h, w = cif.shape
    C, _, ch, cw = caf.shape
    K = int(n_keypoints if n_keypoints is not None else F)
    p = params if params is not None else default_params()
    n_init = 0
    ia = ii = None
    if initial_annotations is not None and len(initial_annotations):
        ia = np.ascontiguousarray(initial_annotations, dtype=np.float32)
        ii = np.ascontiguousarray(initial_ids, dtype=np.int64)
        n_init = ia.shape[0]
    if cap is None:
        cap = F * h * w + n_init + 1
    out = np.zeros((cap, K, 4), dtype=np.float32)
    ids = np.zeros((cap,), dtype=np.int64)
    H, W = (h - 1) * cif_stride + 1, (w - 1) * cif_stride + 1
    t = {}
    if taps:
        t['cifhr'] = np.zeros((F, H, W), dtype=np.float32)
        t['seeds_f'] = np.zeros((F * h * w,), dtype=np.int64)
        t['seeds_vxys'] = np.zeros((F * h * w, 4), dtype=np.float32)
        t['n_seeds'] = ctypes.c_int64(0)
        t['fwd'] = np.zeros((C, ch * cw, 7), dtype=np.float32)
        t['bwd'] = np.zeros((C, ch * cw, 7), dtype=np.float32)
        t['n_fwd'] = np.zeros((C,), dtype=np.int64)
        t['n_bwd'] = np.zeros((C,), dtype=np.int64)
        t['n_pre_nms'] = ctypes.c_int64(0)
    i64, f32 = ctypes.c_int64, ctypes.c_float
    n = lib().oracle_cifcaf_call(
        _ptr(cif, f32), i64(F), i64(h), i64(w), i64(cif_stride),
        _ptr(caf, f32), i64(C), i64(ch), i64(cw), i64(caf_stride),
        _ptr(skeleton, i64), i64(K),
        _ptr(ia, f32), _ptr(ii, i64), i64(n_init),
        ctypes.byref(p),
        _ptr(out, f32), _ptr(ids, i64), i64(cap),
        _ptr(t.get('cifhr'), f32),
        _ptr(t.get('seeds_f'), i64), _ptr(t.get('seeds_vxys'), f32), i64(F * h * w),
        ctypes.byref(t['n_seeds']) if taps else None,
        _ptr(t.get('fwd'), f32), _ptr(t.get('n_fwd'), i64),
        _ptr(t.get('bwd'), f32), _ptr(t.get('n_bwd'), i64),
        ctypes.byref(t['n_pre_nms']) if taps else None)
    n = int(n)
    assert n <= cap
    if not taps:
        return out[:n].copy(), ids[:n].copy()
    ns = int(t['n_seeds'].value)
    taps_out = {
        'cifhr': t['cifhr'],
        'seeds_f': t['seeds_f'][:ns].copy(), 'seeds_vxys': t['seeds_vxys'][:ns].copy(),
        'fwd': [t['fwd'][c, :t['n_fwd'][c]].copy() for c in range(C)],
        'bwd': [t['bwd'][c, :t['n_bwd'][c]].copy() for c in range(C)],
        'n_pre_nms': int(t['n_pre_nms'].value),
    }
    return out[:n].copy(), ids[:n].copy(), taps_out


def decode_det(field, stride, params=None, max_detections_before_nms=120, taps=False):
    """Oracle equivalent of torch.classes.openpifpaf_decoder.CifDet().call(field, stride) on a FRESH instance
    (csrc/src/cifdet.cpp:24-80).  field [F,6,h,w] float32.  params.seed_threshold plays CifDetSeeds::threshold.
    Returns (categories [N] i64, scores [N] f32, boxes [N,4] f32 (x1,y1,x2,y2)[, taps dict])."""
    field = np.ascontiguousarray(field, dtype=np.float32)
    F, ncomp, h, w = field.shape
    assert ncomp == 6
    p = params if params is not None else default_params()
    cap = F * h * w + 1
    cats = np.zeros((cap,), dtype=np.int64)
    scores = np.zeros((cap,), dtype=np.float32)
    boxes = np.zeros((cap, 4), dtype=np.float32)
    H, W = (h - 1) * stride + 1, (w - 1) * stride + 1
    t = {}
    if taps:
        t['cifhr'] = np.zeros((F, H, W), dtype=np.float32)
        t['seeds_f'] = np.zeros((F * h * w,), dtype=np.int64)
        t['seeds_vxywh'] = np.zeros((F * h * w, 5), dtype=np.float32)
        t['n_seeds'] = ctypes.c_int64(0)
    i64, f32 = ctypes.c_int64, ctypes.c_float
    n = int(lib().oracle_cifdet_call(
        _ptr(field, f32), i64(F), i64(h), i64(w), i64(stride), ctypes.byref(p), i64(max_detections_before_nms),
        _ptr(cats, i64), _ptr(scores, f32), _ptr(boxes, f32), i64(cap),
        _ptr(t.get('cifhr'), f32), _ptr(t.get('seeds_f'), i64), _ptr(t.get('seeds_vxywh'), f32), i64(F * h * w),
        ctypes.byref(t['n_seeds']) if taps else None))
    out = (cats[:n].copy(), scores[:n].copy(), boxes[:n].copy())
    if not taps:
        return out
    ns = int(t['n_seeds'].value)
    return out + ({'cifhr': t['cifhr'], 'seeds_f': t['seeds_f'][:ns].copy(),
                   'seeds_vxywh': t['seeds_vxywh'][:ns].copy()},)


def grow_connection_blend(caf, x, y, s, filter_sigmas=1.0, only_max=False):
    caf = np.ascontiguousarray(caf, dtype=np.float32)
    out = (ctypes.c_double * 4)()
    lib().oracle_grow_connection_blend(
        _ptr(caf, ctypes.c_float), ctypes.c_int64(caf.shape[0]),
        ctypes.c_double(x), ctypes.c_double(y), ctypes.c_double(s),
        ctypes.c_double(filter_sigmas), ctypes.c_int(int(only_max)), out)
    return list(out)


# ---------------------------------------------------------------- compiled reference

_ref_loaded = False

# every static the reference extension exposes (csrc/src/module.cpp:26-32,58,76-117), keyed by the name of the
# matching OracleParams field where there is one, with the reference's defaults (csrc/src/*.cpp)
REF_DEFAULTS = {
    'block_joints': False, 'greedy': False, 'keypoint_threshold': 0.15, 'keypoint_threshold_rel': 0.5,
    'reverse_match': True, 'force_complete': False, 'force_complete_caf_th': 0.001,
    'cifhr_neighbors': 16, 'cifhr_threshold': 0.3, 'cifhr_ablation_skip': False,
    'seed_threshold': 0.2, 'seeds_ablation_nms': False, 'seeds_ablation_no_rescore': False,
    'det_seed_threshold': 0.2, 'caf_score_th': 0.3, 'caf_ablation_no_rescore': False,
    'nms_instance_threshold': 0.15, 'nms_keypoint_threshold': 0.15, 'nms_suppression': 0.00001,
    'max_detections_before_nms': 120,
}
# name -> (torchscript class path, static) of REF_DEFAULTS
_REF_STATICS = {
    'block_joints': ('openpifpaf_decoder.CifCaf', 'block_joints'),
    'greedy': ('openpifpaf_decoder.CifCaf', 'greedy'),
    'keypoint_threshold': ('openpifpaf_decoder.CifCaf', 'keypoint_threshold'),
    'keypoint_threshold_rel': ('openpifpaf_decoder.CifCaf', 'keypoint_threshold_rel'),
    'reverse_match': ('openpifpaf_decoder.CifCaf', 'reverse_match'),
    'force_complete': ('openpifpaf_decoder.CifCaf', 'force_complete'),
    'force_complete_caf_th': ('openpifpaf_decoder.CifCaf', 'force_complete_caf_th'),
    'cifhr_neighbors': ('openpifpaf_decoder_utils.CifHr', 'neighbors'),
    'cifhr_threshold': ('openpifpaf_decoder_utils.CifHr', 'threshold'),
    'cifhr_ablation_skip': ('openpifpaf_decoder_utils.CifHr', 'ablation_skip'),
    'seed_threshold': ('openpifpaf_decoder_utils.CifSeeds', 'threshold'),
    'seeds_ablation_nms': ('openpifpaf_decoder_utils.CifSeeds', 'ablation_nms'),
    'seeds_ablation_no_rescore': ('openpifpaf_decoder_utils.CifSeeds', 'ablation_no_rescore'),
    'det_seed_threshold': ('openpifpaf_decoder_utils.CifDetSeeds', 'threshold'),
    'caf_score_th': ('openpifpaf_decoder_utils.CafScored', 'default_score_th'),
    'caf_ablation_no_rescore': ('openpifpaf_decoder_utils.CafScored', 'ablation_no_rescore'),
    'nms_instance_threshold': ('openpifpaf_decoder_utils.NMSKeypoints', 'instance_threshold'),
    'nms_keypoint_threshold': ('openpifpaf_decoder_utils.NMSKeypoints', 'keypoint_threshold'),
    'nms_suppression': ('openpifpaf_decoder_utils.NMSKeypoints', 'suppression'),
    'max_detections_before_nms': ('openpifpaf_decoder.CifDet', 'max_detections_before_nms'),
}
# a reused reference CifCaf / CifDet runs its n-th call at CifHr revision n, until the call that would reach 10 001
# zeroes the buffer and runs at 0 (src/cif_hr.cpp:115-120)
REVISION_WRAP = 10000


def ref_available():
    return os.path.exists(REF_SO)


def load_ref():
    """Load oracle/_ref/refcpp.so (the unmodified reference decoder) into torch."""
    global _ref_loaded
    import torch
    if not _ref_loaded:
        if not os.path.exists(REF_SO):
            from . import build_ref
            build_ref.build()
        torch.ops.load_library(REF_SO)
        torch.ops.openpifpaf.set_quiet(True)
        _ref_loaded = True
    return torch.classes.openpifpaf_decoder


def ref_configure(**kw):
    """Set every reference static (module.cpp:26-32,58,76-117) to `kw` (keys of REF_DEFAULTS) or, when not given,
    back to its default.  The statics are process-global: without the reset, one call's options would leak into
    every later reference run of the process."""
    import torch
    load_ref()
    unknown = set(kw) - set(REF_DEFAULTS)
    assert not unknown, f'not a reference static: {sorted(unknown)}'
    for k, default in REF_DEFAULTS.items():
        path, static = _REF_STATICS[k]
        ns, cls = path.split('.')
        getattr(getattr(getattr(torch.classes, ns), cls), 'set_' + static)(type(default)(kw.get(k, default)))


def ref_statics():
    """the current value of every reference static, keyed like REF_DEFAULTS"""
    import torch
    load_ref()
    out = {}
    for k, (path, static) in _REF_STATICS.items():
        ns, cls = path.split('.')
        out[k] = getattr(getattr(getattr(torch.classes, ns), cls), 'get_' + static)()
    return out


def calls_before(revision):
    """calls a reused reference instance makes before the call that runs at CifHr `revision`"""
    assert revision == int(revision) and 0 <= revision <= REVISION_WRAP, revision
    return REVISION_WRAP if revision == 0 else int(revision) - 1


def _advance(revisions, zero_call):
    """yield once before each call of an instance that runs at the next of `revisions`, after making the calls before it
    on all-zero fields (calls_before).  With a CifHr threshold above 0 those write nothing, so the map stays as clean
    as a fresh one: zeroed at the wrap to revision 0, where a never-written pixel reads 0 (src/cif_seeds.cpp:17-30),
    and -1 at every other revision.  Pixels an earlier decode of the sequence wrote hold at most its revision + 1, so
    they read -1 from two revisions on; a sequence may not decode at two consecutive revisions."""
    import torch
    calls, last = 0, None
    for r in revisions:
        n = calls_before(r)
        assert n >= calls, f'revisions out of call order: {list(revisions)}'
        assert last is None or r == 0 or r > last + 1, f'revision {r} right after {last} reads a dirty map'
        if n > calls:
            assert torch.classes.openpifpaf_decoder_utils.CifHr.get_threshold() > 0.0, \
                'zero fields write the CifHr map at threshold 0'
        for _ in range(n - calls):
            zero_call()
        yield r
        calls, last = n + 1, r


def ref_decode(cif, cif_stride, caf, caf_stride, skeleton, n_keypoints=None,
               initial_annotations=None, initial_ids=None, taps=False, revision=1):
    """Run the unmodified reference on a CifCaf instance that decodes at CifHr `revision` (integer, 0 to
    REVISION_WRAP; 1 = a FRESH instance).  See ref_decode_revisions."""
    return ref_decode_revisions(cif, cif_stride, caf, caf_stride, skeleton, n_keypoints, initial_annotations,
                                initial_ids, taps, revisions=(revision,))[0]


def ref_decode_revisions(cif, cif_stride, caf, caf_stride, skeleton, n_keypoints=None,
                         initial_annotations=None, initial_ids=None, taps=False, revisions=(1,)):
    """The same decode on ONE reference CifCaf instance at each of `revisions` (in call order: 1, 2, ..., 10000,
    then 0), the calls in between made on all-zero fields of the same shape (_advance).  Returns a list of what
    ref_decode returns."""
    import torch
    dec = load_ref()
    cif_t = torch.from_numpy(np.ascontiguousarray(cif, dtype=np.float32))
    caf_t = torch.from_numpy(np.ascontiguousarray(caf, dtype=np.float32))
    sk = torch.from_numpy(np.ascontiguousarray(skeleton, dtype=np.int64))
    K = int(n_keypoints if n_keypoints is not None else cif_t.shape[0])
    inst = dec.CifCaf(K, sk)
    zc, zf = torch.zeros_like(cif_t), torch.zeros_like(caf_t)
    out = []
    for _ in _advance(revisions, lambda: inst.call(zc, cif_stride, zf, caf_stride)):
        out.append(_ref_cifcaf_call(inst, cif_t, cif_stride, caf_t, caf_stride, sk, initial_annotations,
                                    initial_ids, taps))
    return out


def _ref_cifcaf_call(inst, cif_t, cif_stride, caf_t, caf_stride, sk, initial_annotations, initial_ids, taps):
    import torch
    ia = ii = None
    if initial_annotations is not None and len(initial_annotations):
        ia = torch.from_numpy(np.ascontiguousarray(initial_annotations, dtype=np.float32))
        ii = torch.from_numpy(np.ascontiguousarray(initial_ids, dtype=np.int64))
    ann, ids = inst.call_with_initial_annotations(cif_t, cif_stride, caf_t, caf_stride, ia, ii)
    if not taps:
        return ann.numpy().copy(), ids.numpy().copy()
    u = torch.classes.openpifpaf_decoder_utils
    hr, rev = inst.get_cifhr()
    hr = hr.clone()
    seeds = u.CifSeeds(hr, rev)
    seeds.fill(cif_t, cif_stride)
    sf, sv = seeds.get()
    cs = u.CafScored(hr, rev, -1.0, 0.1)
    cs.fill(caf_t, caf_stride, sk)
    fwd, bwd = cs.get()
    t = {'cifhr': hr.numpy().copy(), 'revision': float(rev),
         'seeds_f': sf.numpy().copy(), 'seeds_vxys': sv.numpy().copy(),
         'fwd': [x.clone().numpy() for x in fwd], 'bwd': [x.clone().numpy() for x in bwd]}
    return ann.numpy().copy(), ids.numpy().copy(), t


def ref_decode_det(field, stride, revision=1):
    """Run the unmodified reference CifDet (csrc/src/cifdet.cpp) on an instance that decodes at CifHr `revision`
    (1 = a FRESH instance; see ref_decode_det_revisions)."""
    return ref_decode_det_revisions(field, stride, (revision,))[0]


def ref_decode_det_revisions(field, stride, revisions=(1,)):
    """ref_decode_revisions for CifDet.  (CifDetHr is not exported as a TorchScript class, module.cpp:76-102, so
    there are no stage taps on this side.)"""
    import torch
    dec = load_ref()
    f_t = torch.from_numpy(np.ascontiguousarray(field, dtype=np.float32))
    inst = dec.CifDet()
    zero = torch.zeros_like(f_t)
    out = []
    for _ in _advance(revisions, lambda: inst.call(zero, stride)):
        cats, scores, boxes = inst.call(f_t, stride)
        out.append((cats.numpy().copy(), scores.numpy().copy(), boxes.numpy().copy().reshape(-1, 4)))
    return out
