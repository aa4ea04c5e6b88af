"""Host-side mirror of the reference decoder operator surface, backed by libpifpaf_b200.

Reference interface (paths relative to the reference's src/openpifpaf/):
  torch.classes.openpifpaf_decoder.CifCaf          csrc/src/module.cpp:24-58
  torch.classes.openpifpaf_decoder_utils.{CifHr,CifSeeds,CafScored,NMSKeypoints}
                                                   csrc/src/module.cpp:66-118
  torch.ops.openpifpaf_decoder.grow_connection_blend   csrc/src/module.cpp:60

Same names, argument meaning, return types and error behaviour (RuntimeError);
the static get_/set_ pairs configure class attributes that are snapshotted BY
VALUE into every native call.  Extra, beyond the reference: `decode_batch()` on
device-resident field batches (fields never visit the host).
"""
import ctypes

import numpy as np
import torch

from . import _lib


def _static(name, default):
    """reference STATIC_GETSET macro (csrc/src/module.cpp:16)"""
    def getter(cls):
        return getattr(cls, '_' + name)

    def setter(cls, v):
        setattr(cls, '_' + name, type(default)(v))
    return default, classmethod(getter), classmethod(setter)


class _Statics(type):
    """Metaclass turning `STATICS = {name: default}` into _name / get_name / set_name."""
    def __new__(mcs, clsname, bases, ns):
        for name, default in ns.get('STATICS', {}).items():
            d, g, s = _static(name, default)
            ns['_' + name] = d
            ns['get_' + name] = g
            ns['set_' + name] = s
        return super().__new__(mcs, clsname, bases, ns)


class CifHr(metaclass=_Statics):
    """statics of csrc/src/cif_hr.cpp:13-15"""
    STATICS = {'neighbors': 16, 'threshold': 0.3, 'ablation_skip': False}


class CifSeeds(metaclass=_Statics):
    """statics of csrc/src/cif_seeds.cpp:11-14"""
    STATICS = {'threshold': 0.2, 'ablation_nms': False, 'ablation_no_rescore': False}


class CafScored(metaclass=_Statics):
    """statics of csrc/src/caf_scored.cpp:11-12"""
    STATICS = {'default_score_th': 0.3, 'ablation_no_rescore': False}


class NMSKeypoints(metaclass=_Statics):
    """statics of csrc/src/nms_keypoints.cpp:12-14"""
    STATICS = {'suppression': 0.00001, 'instance_threshold': 0.15, 'keypoint_threshold': 0.15}


def _as_f32_cpu(t, name):
    if isinstance(t, np.ndarray):
        t = torch.from_numpy(t)
    if not isinstance(t, torch.Tensor):
        raise RuntimeError(f'{name} must be a tensor')
    if t.dtype != torch.float32:
        raise RuntimeError(f'{name} must be of type float32')     # accessor<float, 4> in the reference
    return t


class CifCaf(metaclass=_Statics):
    """Drop-in for torch.classes.openpifpaf_decoder.CifCaf (csrc/include/openpifpaf/decoder/cifcaf.hpp:79-145).

    :param n_keypoints: number of keypoints K
    :param skeleton: LongTensor [C, 2], 0-based (decoder/cifcaf.py:119-122 passes ``skeleton - 1``)
    """
    STATICS = {
        'block_joints': False, 'greedy': False,
        'keypoint_threshold': 0.15, 'keypoint_threshold_rel': 0.5,
        'reverse_match': True, 'force_complete': False, 'force_complete_caf_th': 0.001,
    }
    #: per-image capacity for annotations before NMS.  The reference grows a std::vector; here an image that needs
    #: more raises RuntimeError (PIFPAF_E_OVERFLOW) from fetch -- raise this attribute before the first decode then.
    max_annotations = 512

    def __init__(self, n_keypoints, skeleton, *, device=0, n_cif_fields=None):
        if isinstance(skeleton, np.ndarray):
            skeleton = torch.from_numpy(skeleton)
        if not isinstance(skeleton, torch.Tensor) or skeleton.dtype != torch.int64:
            raise RuntimeError('skeleton must be of type LongTensor')     # cifcaf.hpp:106
        self.n_keypoints = int(n_keypoints)
        self.skeleton = skeleton.detach().cpu().contiguous().reshape(-1, 2)
        self.n_cif_fields = int(n_cif_fields) if n_cif_fields is not None else self.n_keypoints
        self.device = int(device)
        self._handle = None
        self._caps = None
        self.last_revision = 1.0

    # --- pickling: state is (n_keypoints, skeleton) like csrc/src/module.cpp:40-55
    def __getstate__(self):
        return (self.n_keypoints, self.skeleton, self.device, self.n_cif_fields)

    def __setstate__(self, state):
        n_keypoints, skeleton, device, n_cif_fields = state
        self.__init__(n_keypoints, skeleton, device=device, n_cif_fields=n_cif_fields)

    def __del__(self):
        self._free()

    def _free(self):
        h, self._handle = getattr(self, '_handle', None), None
        if h is not None:
            try:
                _lib.lib().pifpaf_decoder_destroy(h)
            except Exception:   # interpreter shutdown
                pass

    # --- native handle with capacities that only ever grow
    def reserve(self, batch, h, w, stride):
        """Size the native workspace up front (e.g. from a compiled net's max batch and head shape) so that it is
        never re-created while results are in flight."""
        self._ensure(int(batch), int(h), int(w), int(stride))

    def _ensure(self, batch, h, w, stride):
        caps = self._caps
        need = (batch, h, w, stride, self.max_annotations)
        if caps is not None and all(c >= n for c, n in zip(caps, need)):
            return self._handle
        if getattr(self, '_begun', None):
            # re-creating the handle would free the pinned result buffers and events of fetches in flight
            raise RuntimeError('decoder capacity exceeded while results are pending: fetch_end() them first, or '
                               'reserve() the largest batch / field shape before pipelining')
        if caps is not None:
            need = tuple(max(c, n) for c, n in zip(caps, need))
        self._free()
        handle = ctypes.c_void_p()
        sk = self.skeleton.numpy()
        _lib.check(_lib.lib().pifpaf_decoder_create(
            ctypes.byref(handle), self.device, self.n_keypoints, self.n_cif_fields, sk.shape[0],
            sk.ctypes.data_as(ctypes.c_void_p), need[0], need[1], need[2], need[3], need[4]))
        self._handle, self._caps = handle, need
        return handle

    @classmethod
    def params(cls, **overrides):
        """Snapshot the reference-style statics into a by-value params struct."""
        p = _lib.default_params(
            cifhr_neighbors=CifHr._neighbors, cifhr_threshold=CifHr._threshold,
            cifhr_ablation_skip=int(CifHr._ablation_skip),
            seed_threshold=CifSeeds._threshold, seeds_ablation_nms=int(CifSeeds._ablation_nms),
            seeds_ablation_no_rescore=int(CifSeeds._ablation_no_rescore),
            caf_score_th=CafScored._default_score_th,
            caf_ablation_no_rescore=int(CafScored._ablation_no_rescore),
            block_joints=int(cls._block_joints), greedy=int(cls._greedy),
            keypoint_threshold=cls._keypoint_threshold, keypoint_threshold_rel=cls._keypoint_threshold_rel,
            reverse_match=int(cls._reverse_match), force_complete=int(cls._force_complete),
            force_complete_caf_th=cls._force_complete_caf_th,
            nms_suppression=NMSKeypoints._suppression, nms_instance_threshold=NMSKeypoints._instance_threshold,
            nms_keypoint_threshold=NMSKeypoints._keypoint_threshold)
        for k, v in overrides.items():
            setattr(p, k, v)
        return p

    # --- reference methods
    def call(self, cif_field, cif_stride, caf_field, caf_stride):
        """csrc/src/cifcaf.cpp:116-123"""
        return self.call_with_initial_annotations(cif_field, cif_stride, caf_field, caf_stride, None, None)

    def call_with_initial_annotations(self, cif_field, cif_stride, caf_field, caf_stride,
                                      initial_annotations=None, initial_ids=None):
        """csrc/src/cifcaf.cpp:126-262.  cif_field [F,5,h,w], caf_field [C,8,h,w] float32 (CPU or CUDA);
        returns (annotations [N,K,4] (v,x,y,s) float32 CPU, ids [N] int64 CPU)."""
        cif_field = _as_f32_cpu(cif_field, 'cif_field')
        caf_field = _as_f32_cpu(caf_field, 'caf_field')
        if cif_field.dim() != 4 or caf_field.dim() != 4 or cif_field.shape[1] < 5 or caf_field.shape[1] < 8:
            raise RuntimeError('expected cif_field [F,5,h,w] and caf_field [C,8,h,w]')
        if cif_field.shape[0] != self.n_cif_fields or caf_field.shape[0] != self.skeleton.shape[0]:
            raise RuntimeError('field count does not match n_keypoints / skeleton')
        if cif_field.shape[2:] != caf_field.shape[2:]:
            raise RuntimeError('cif and caf fields must have the same spatial shape')
        if initial_annotations is not None and initial_ids is None:
            raise RuntimeError('require initial_ids when initial_annotations are given')   # cifcaf.cpp:178
        h, w = int(cif_field.shape[2]), int(cif_field.shape[3])
        K = self.n_keypoints
        p = self.params()
        self.last_revision = p.cifhr_revision
        self.set_tap_shape(h, w, int(cif_stride))

        if cif_field.is_cuda or caf_field.is_cuda:
            init = None
            if initial_annotations is not None and len(initial_annotations):
                init = (initial_annotations.reshape(1, -1, K, 4), initial_ids.reshape(1, -1))
            res = self.decode_batch(cif_field[:, :5].unsqueeze(0), int(cif_stride),
                                    caf_field[:, :8].unsqueeze(0), int(caf_stride), initial=init)
            return res[0]

        handle = self._ensure(1, h, w, max(int(cif_stride), int(caf_stride)))
        cif_c = cif_field[:, :5].contiguous()
        caf_c = caf_field[:, :8].contiguous()
        n_init = 0
        ia_ptr = ii_ptr = None
        if initial_annotations is not None and len(initial_annotations):
            ia = _as_f32_cpu(initial_annotations, 'initial_annotations').contiguous()
            ii = initial_ids.to(torch.int64).contiguous()
            n_init = int(ia.shape[0])
            ia_ptr, ii_ptr = ia.data_ptr(), ii.data_ptr()
        cap = self.max_annotations
        out = torch.empty((cap, K, 4), dtype=torch.float32)
        ids = torch.empty((cap,), dtype=torch.int64)
        n = ctypes.c_int32(0)
        _lib.check(_lib.lib().pifpaf_decoder_call(
            handle, cif_c.data_ptr(), int(cif_stride), caf_c.data_ptr(), int(caf_stride), h, w,
            ia_ptr, ii_ptr, n_init, ctypes.byref(p), out.data_ptr(), ids.data_ptr(), cap, ctypes.byref(n)))
        return out[:n.value].clone(), ids[:n.value].clone()

    def decode_batch(self, cif_batch, cif_stride, caf_batch, caf_stride, *, initial=None, stream=None):
        """Batched decode of device-resident fields: cif_batch [B,F,5,h,w], caf_batch [B,C,8,h,w]
        CUDA float32.  Returns a list of B (annotations [N,K,4], ids [N]) CPU tensor pairs."""
        self.decode_batch_async(cif_batch, cif_stride, caf_batch, caf_stride, initial=initial, stream=stream)
        return self.fetch(stream=stream)

    def decode_batch_async(self, cif_batch, cif_stride, caf_batch, caf_stride, *, initial=None, stream=None):
        if not (cif_batch.is_cuda and caf_batch.is_cuda):
            raise RuntimeError('decode_batch expects CUDA tensors (use call() for host fields)')
        if cif_batch.dtype != torch.float32 or caf_batch.dtype != torch.float32:
            raise RuntimeError('fields must be of type float32')
        cif_batch = cif_batch.contiguous()
        caf_batch = caf_batch.contiguous()
        B, F, ncomp, h, w = cif_batch.shape
        if ncomp != 5 or caf_batch.shape[2] != 8 or F != self.n_cif_fields \
                or caf_batch.shape[1] != self.skeleton.shape[0] or caf_batch.shape[0] != B \
                or tuple(caf_batch.shape[3:]) != (h, w):
            raise RuntimeError('expected cif [B,F,5,h,w] and caf [B,C,8,h,w]')
        if cif_batch.device.index != self.device or caf_batch.device.index != self.device:
            raise RuntimeError('fields live on a different CUDA device than the decoder')
        handle = self._ensure(int(B), int(h), int(w), max(int(cif_stride), int(caf_stride)))
        p = self.params()
        self.last_revision = p.cifhr_revision
        self.set_tap_shape(int(h), int(w), int(cif_stride))
        ia_ptr = ii_ptr = ic_ptr = None
        init_cap = 0
        if initial is not None:
            ia, ii = initial
            ia = ia.to(device=cif_batch.device, dtype=torch.float32).contiguous()
            ii = ii.to(device=cif_batch.device, dtype=torch.int64).contiguous()
            counts = torch.full((B,), ia.shape[1], dtype=torch.int32, device=cif_batch.device)
            init_cap = int(ia.shape[1])
            ia_ptr, ii_ptr, ic_ptr = ia.data_ptr(), ii.data_ptr(), counts.data_ptr()
            self._keepalive = (ia, ii, counts)
        st = stream if stream is not None else torch.cuda.current_stream(cif_batch.device)
        self._keepalive_fields = (cif_batch, caf_batch)
        self._last_batch = int(B)
        _lib.check(_lib.lib().pifpaf_decoder_decode_device(
            handle, cif_batch.data_ptr(), caf_batch.data_ptr(), int(B), int(h), int(w),
            int(cif_stride), int(caf_stride), ia_ptr, ii_ptr, ic_ptr, init_cap,
            ctypes.byref(p), ctypes.c_void_p(st.cuda_stream)))

    def fetch(self, *, stream=None):
        """Wait for the last decode_batch_async and return its per-image results."""
        self.fetch_begin(stream=stream)
        return self.fetch_end()

    def fetch_begin(self, *, stream=None):
        """Enqueue the (single, small) async D2H of the last decode's packed results; pair with fetch_end().
        A further decode_batch_async may be enqueued in between (results are double buffered)."""
        st = stream if stream is not None else torch.cuda.current_stream(self.device)
        _lib.check(_lib.lib().pifpaf_decoder_fetch_begin(self._handle, ctypes.c_void_p(st.cuda_stream)))
        self._begun = getattr(self, '_begun', [])
        self._begun.append(self._last_batch)

    def fetch_end(self):
        B, K = self._begun.pop(0), self.n_keypoints
        counts = np.zeros((B,), dtype=np.int32)
        _lib.check(_lib.lib().pifpaf_decoder_fetch_peek(self._handle, counts.ctypes.data))
        cap = max(int(counts.max()) if B else 0, 1)
        ann = np.empty((B, cap, K, 4), dtype=np.float32)
        ids = np.empty((B, cap), dtype=np.int64)
        _lib.check(_lib.lib().pifpaf_decoder_fetch_end(
            self._handle, counts.ctypes.data, ann.ctypes.data, ids.ctypes.data, cap))
        return [(torch.from_numpy(ann[b, :counts[b]].copy()), torch.from_numpy(ids[b, :counts[b]].copy()))
                for b in range(B)]

    def last_stats(self):
        """Work counters of the last decode over its batch (synchronises): hi-res pixels written, seeds, CAF list
        entries, annotations before NMS."""
        out = (ctypes.c_int64 * 10)()
        _lib.check(_lib.lib().pifpaf_decoder_last_stats(self._handle, out, 10))
        return {'cifhr_pixels_written': int(out[0]), 'seeds': int(out[1]), 'caf_entries': int(out[2]),
                'annotations_before_nms': int(out[3]), 'grow_rounds': int(out[4]), 'grow_seeds_grown': int(out[5]),
                'grow_clocks': {'setup': int(out[6]), 'select': int(out[7]), 'grow': int(out[8]), 'commit': int(out[9])}}

    def get_cifhr(self, image=0):
        """csrc/src/module.cpp:36-38: (accumulated [F,H,W] float32, revision)."""
        if self._handle is None:
            raise RuntimeError('no decode yet')
        return self.tap_cifhr(image), self.last_revision

    # --- stage taps (parity tests; the reference exposes the same stages through decoder_utils classes)
    def tap_cifhr(self, image=0):
        F = self.n_cif_fields
        H, W = self._tap_shape
        out = np.empty((F, H, W), dtype=np.float32)
        _lib.check(_lib.lib().pifpaf_decoder_tap_cifhr(self._handle, image, out.ctypes.data, out.size))
        return torch.from_numpy(out)

    def tap_seeds(self, image=0):
        cap = self.n_cif_fields * self._tap_hw
        f = np.empty((cap,), dtype=np.int64)
        vxys = np.empty((cap, 4), dtype=np.float32)
        n = ctypes.c_int64(0)
        _lib.check(_lib.lib().pifpaf_decoder_tap_seeds(self._handle, image, f.ctypes.data, vxys.ctypes.data,
                                                       cap, ctypes.byref(n)))
        return torch.from_numpy(f[:n.value].copy()), torch.from_numpy(vxys[:n.value].copy())

    def tap_caf(self, image=0):
        C, hw = self.skeleton.shape[0], self._tap_hw
        fwd = np.empty((C, hw, 7), dtype=np.float32)
        bwd = np.empty((C, hw, 7), dtype=np.float32)
        nf = np.zeros((C,), dtype=np.int64)
        nb = np.zeros((C,), dtype=np.int64)
        _lib.check(_lib.lib().pifpaf_decoder_tap_caf(self._handle, image, fwd.ctypes.data, nf.ctypes.data,
                                                     bwd.ctypes.data, nb.ctypes.data))
        return ([torch.from_numpy(fwd[c, :nf[c]].copy()) for c in range(C)],
                [torch.from_numpy(bwd[c, :nb[c]].copy()) for c in range(C)])

    def set_tap_shape(self, h, w, stride):
        """Field shape of the decode whose stages are tapped."""
        self._tap_shape = ((h - 1) * stride + 1, (w - 1) * stride + 1)
        self._tap_hw = h * w


class CifDetSeeds(metaclass=_Statics):
    """static of csrc/src/cif_seeds.cpp:12 (module.cpp:96-97)"""
    STATICS = {'threshold': 0.2}


class CifDet(metaclass=_Statics):
    """Drop-in for torch.classes.openpifpaf_decoder.CifDet (csrc/include/openpifpaf/decoder/cifdet.hpp:33-47,
    csrc/src/cifdet.cpp:24-80): ``call(cifdet_field [F,6,h,w], stride) -> (categories [N] int64 (1-based),
    scores [N] float32, boxes [N,4] float32 (x1, y1, x2, y2))`` -- before NMS, like the reference class; the statics
    CifHr.{neighbors,threshold}, CifDetSeeds.threshold and max_detections_before_nms go by value into every call.
    Beyond the reference: ``decode_batch`` on device-resident field batches, optionally with the NMS / score filter
    of the reference's Python wrapper (decoder/cifdet.py:55-64) done on the GPU."""
    STATICS = {'max_detections_before_nms': 120}
    #: capacity of the native handle for max_detections_before_nms
    max_detections = 1024

    def __init__(self, n_categories=None, *, device=0):
        self.n_categories = None if n_categories is None else int(n_categories)
        self.device = int(device)
        self._handle = None
        self._caps = None
        self._pending = None

    def __getstate__(self):
        return (self.n_categories, self.device)

    def __setstate__(self, state):
        self.__init__(state[0], device=state[1])

    def __del__(self):
        self._free()

    def _free(self):
        h, self._handle = getattr(self, '_handle', None), None
        if h is not None:
            try:
                _lib.lib().pifpaf_cifdet_destroy(h)
            except Exception:   # interpreter shutdown
                pass

    def _ensure(self, n_categories, batch, h, w, stride):
        if self.n_categories is None:
            self.n_categories = int(n_categories)
        if int(n_categories) != self.n_categories:
            raise RuntimeError('field count does not match the number of categories of this decoder')
        need = (batch, h, w, stride, max(self.max_detections, self._max_detections_before_nms))
        if self._caps is not None and all(c >= n for c, n in zip(self._caps, need)):
            return self._handle
        if self._caps is not None:
            need = tuple(max(c, n) for c, n in zip(self._caps, need))
        self._free()
        handle = ctypes.c_void_p()
        _lib.check(_lib.lib().pifpaf_cifdet_create(ctypes.byref(handle), self.device, self.n_categories, *need))
        self._handle, self._caps = handle, need
        return handle

    @classmethod
    def params(cls, **overrides):
        p = _lib.CifDetParams()
        _lib.check(_lib.lib().pifpaf_cifdet_default_params(ctypes.byref(p)))
        p.cifhr_neighbors, p.cifhr_threshold = CifHr._neighbors, CifHr._threshold
        p.seed_threshold = CifDetSeeds._threshold
        p.max_detections_before_nms = cls._max_detections_before_nms
        for k, v in overrides.items():
            if not hasattr(p, k):
                raise AttributeError(f'unknown CifDet parameter {k}')
            setattr(p, k, v)
        return p

    @staticmethod
    def _unpack(rec, n, filtered):
        rec = rec[:n]
        if filtered:
            rec = rec[rec[:, 7] > 0.5]
            scores = rec[:, 6]
        else:
            scores = rec[:, 1]
        return (torch.from_numpy(rec[:, 0].astype(np.int64)), torch.from_numpy(scores.copy()),
                torch.from_numpy(rec[:, 2:6].copy()))

    def call(self, cifdet_field, cifdet_stride):
        """csrc/src/cifdet.cpp:24-80"""
        field = _as_f32_cpu(cifdet_field, 'cifdet_field')
        if field.dim() != 4 or field.shape[1] < 6:
            raise RuntimeError('expected cifdet_field [F,6,h,w]')
        if field.is_cuda:
            return self.decode_batch(field[:, :6].unsqueeze(0), int(cifdet_stride))[0]
        F, _, h, w = (int(v) for v in field.shape)
        handle = self._ensure(F, 1, h, w, int(cifdet_stride))
        p = self.params()
        cap = int(p.max_detections_before_nms)
        rec = np.empty((cap, 8), dtype=np.float32)
        n = ctypes.c_int32(0)
        fc = field[:, :6].contiguous()
        _lib.check(_lib.lib().pifpaf_cifdet_call(handle, fc.data_ptr(), int(cifdet_stride), h, w, ctypes.byref(p),
                                                 rec.ctypes.data, cap, ctypes.byref(n)))
        return self._unpack(rec, n.value, False)

    def decode_batch(self, field_batch, stride, *, nms=False, iou_threshold=0.5, nms_by_category=True,
                     suppression=0.1, instance_threshold=0.15, stream=None):
        """field_batch [B,F,6,h,w] CUDA float32.  nms=False: per image the raw (categories, scores, boxes) of
        CifDet::call; nms=True: the filtered detections of decoder/cifdet.py:55-64 (scores after suppression)."""
        self.decode_batch_async(field_batch, stride, nms=nms, iou_threshold=iou_threshold,
                                nms_by_category=nms_by_category, suppression=suppression,
                                instance_threshold=instance_threshold, stream=stream)
        return self.fetch(stream=stream)

    def decode_batch_async(self, field_batch, stride, *, nms=False, iou_threshold=0.5, nms_by_category=True,
                           suppression=0.1, instance_threshold=0.15, stream=None):
        """Enqueue the decode of decode_batch on `stream` (default: the current stream of the fields' device) without
        waiting for it; fetch() returns its results."""
        if not field_batch.is_cuda or field_batch.dtype != torch.float32:
            raise RuntimeError('decode_batch expects a CUDA float32 tensor (use call() for host fields)')
        field_batch = field_batch.contiguous()
        B, F, ncomp, h, w = (int(v) for v in field_batch.shape)
        if ncomp != 6:
            raise RuntimeError('expected cifdet fields [B,F,6,h,w]')
        if field_batch.device.index != self.device:
            raise RuntimeError('fields live on a different CUDA device than the decoder')
        handle = self._ensure(F, B, h, w, int(stride))
        p = self.params(nms=int(bool(nms)), iou_threshold=float(iou_threshold), nms_by_category=int(bool(nms_by_category)),
                        suppression=float(suppression), instance_threshold=float(instance_threshold))
        st = stream if stream is not None else torch.cuda.current_stream(field_batch.device)
        _lib.check(_lib.lib().pifpaf_cifdet_decode_device(handle, field_batch.data_ptr(), B, h, w, int(stride),
                                                          ctypes.byref(p), ctypes.c_void_p(st.cuda_stream)))
        self._pending = (B, int(p.max_detections_before_nms), bool(nms))

    def fetch(self, *, stream=None):
        """Results of the last decode_batch_async, copied back on `stream` (default: the current stream of the
        decoder's device; give the stream the decode was enqueued on): per image (categories, scores, boxes)."""
        pending, self._pending = getattr(self, '_pending', None), None
        if pending is None:
            raise RuntimeError('fetch() without a preceding decode_batch_async()')
        B, cap, nms = pending
        st = stream if stream is not None else torch.cuda.current_stream(self.device)
        counts = np.zeros((B,), dtype=np.int32)
        rec = np.empty((B, cap, 8), dtype=np.float32)
        _lib.check(_lib.lib().pifpaf_cifdet_fetch(self._handle, counts.ctypes.data, rec.ctypes.data, cap,
                                                  ctypes.c_void_p(st.cuda_stream)))
        return [self._unpack(rec[b], int(counts[b]), nms) for b in range(B)]


def grow_connection_blend(caf, x, y, s, filter_sigmas=1.0, only_max=False):
    """torch.ops.openpifpaf_decoder.grow_connection_blend (csrc/src/cifcaf.cpp:105-113): returns [x, y, s, v]."""
    caf = _as_f32_cpu(caf, 'caf').contiguous()
    out = (ctypes.c_double * 4)()
    _lib.check(_lib.lib().pifpaf_grow_connection_blend(
        caf.data_ptr(), int(caf.shape[0]), float(x), float(y), float(s), float(filter_sigmas),
        int(bool(only_max)), out))
    return list(out)
