"""Decoder plugin for the reference framework (imported only from ``register()``, i.e. only when the
reference package ``openpifpaf`` is installed and is importing its plugins).

Reference interfaces implemented (paths relative to the reference's src/openpifpaf/):
  Decoder.cli / configure / factory / __call__ / batch     decoder/decoder.py:21-145
  CifCaf (the decoder this one replaces)                   decoder/cifcaf.py:81-277
  decoder selection by priority                            decoder/factory.py:110-160

Two levels of drop-in:
  * ``CifCafB200.__call__(fields)``: same contract as ``CifCaf.__call__`` (fields of one image, CPU or CUDA
    tensors) -> ``List[Annotation]``; decoding happens on the GPU through libpifpaf_b200.
  * ``CifCafB200.batch(model, image_batch, device=...)``: the whole hot loop on the GPU -- the model is
    compiled once per input shape into wgmma kernels and the head tensors never visit the host.
    ``CifDetB200.batch`` does the same for detection models (one CifDet head); a model the compiled forward does
    not implement (network.UnsupportedModel, e.g. MobileNetV3) takes the reference's ``Decoder.batch`` instead.
    ``register()`` makes ``Multi.batch`` (what ``Predictor`` calls, predictor.py:131) delegate to either when
    it is the only decoder.
"""
import collections
import logging
import time
import weakref

import numpy as np
import torch

from . import decoder as b200_decoder
from . import network as b200_network
from . import predictor as b200_predictor

LOG = logging.getLogger(__name__)


class _CompileCache:
    """The compiled models of the GPU batch path (CifCafB200.batch, CifDetB200.batch): an LRU of
    `compile_cache_size` predictors keyed by (model, input shape); the class using it sets ``self._compiled`` to an
    OrderedDict and implements ``_compile(shell, h, w, batch, device_index)``."""
    #: compiled (model, input shape) entries kept alive; each owns every activation buffer of its max batch
    compile_cache_size = 2

    @staticmethod
    def _weights_version(shell):
        # torch bumps Tensor._version on every in-place write (optimizer step, load_state_dict, .copy_)
        return sum(int(p._version) for p in shell.parameters()) + sum(int(b._version) for b in shell.buffers())

    def _predictor_for(self, shell, batch, h, w, device):
        """Compile `shell` for this input shape once; LRU of `compile_cache_size` entries.  An entry is reused only
        for the same live module object (weak reference, so a recycled id() cannot alias), unchanged weights and a
        batch that fits; evicted entries free their GPU buffers at once."""
        key = (id(shell), h, w)
        hit = self._compiled.get(key)
        if hit is not None:
            ref, version, pred = hit
            if ref() is shell and version == self._weights_version(shell) and pred.net.max_batch >= batch:
                self._compiled.move_to_end(key)
                return pred
            self._evict(key)
        dev_index = torch.device(device).index if device is not None else None
        if dev_index is None:
            dev_index = torch.cuda.current_device()
        pred = self._compile(shell, h, w, max(batch, 1), dev_index)
        self._compiled[key] = (weakref.ref(shell), self._weights_version(shell), pred)
        while len(self._compiled) > self.compile_cache_size:
            self._evict(next(iter(self._compiled)))
        return pred

    def _evict(self, key):
        _, _, pred = self._compiled.pop(key)
        pred.close()


def _build_class():
    import openpifpaf
    from openpifpaf import headmeta
    from openpifpaf.annotation import Annotation
    from openpifpaf.decoder import Decoder

    class CifCafB200(_CompileCache, Decoder):
        """CifCaf decoding on an H100 (same CLI knobs as the reference's CifCaf)."""
        fast_batch = True
        #: read by TrackingPose.soft_nms (tracking_pose.py:160) when this class is its pose generator
        occupancy_visualizer = None

        def __init__(self, cif_metas, caf_metas):
            super().__init__()
            self.cif_metas = cif_metas
            self.caf_metas = caf_metas
            self.score_weights = cif_metas[0].score_weights
            self.native = b200_decoder.CifCaf(
                len(cif_metas[0].keypoints),
                torch.LongTensor(caf_metas[0].skeleton) - 1,          # decoder/cifcaf.py:119-122
            )
            # outrank the reference's CPU CifCaf (decoder/cifcaf.py:123-125 uses the same base + n_fields/1000)
            self.priority += 1.0
            self.priority += sum(m.n_fields for m in cif_metas) / 1000.0
            self.priority += sum(m.n_fields for m in caf_metas) / 1000.0
            self._compiled = collections.OrderedDict()

        @classmethod
        def cli(cls, parser):
            group = parser.add_argument_group('CifCafB200 decoder')
            group.add_argument('--b200-no-fast-batch', dest='b200_fast_batch', default=True, action='store_false',
                               help='decode on the GPU but keep the reference model forward / host transfer')
            group.add_argument('--b200-compile-cache', type=int, default=cls.compile_cache_size,
                               help='number of (model, input shape) compilations kept on the GPU')

        @classmethod
        def configure(cls, args):
            """Only this plugin's own flags.  Every decoding knob (thresholds, force-complete, greedy, ablations) is
            owned by the reference: its CifCaf.configure / decoder.factory.configure (decoder/cifcaf.py:174-211,
            decoder/factory.py:52-82) write the C++ statics of the reference extension, and `sync_statics` reads
            them back before every decode -- one source of truth, independent of the order in which the members
            of the DECODERS set are configured (CifCaf.configure mutates the argparse namespace)."""
            cls.fast_batch = getattr(args, 'b200_fast_batch', True)
            cls.compile_cache_size = max(1, int(getattr(args, 'b200_compile_cache', cls.compile_cache_size)))

        @classmethod
        def sync_statics(cls):
            """Snapshot the reference's process-global statics (csrc/src/module.cpp:26-32,76-117) into the native
            decoder's statics; they go by value into every native call."""
            ref = torch.classes.openpifpaf_decoder.CifCaf
            utl = torch.classes.openpifpaf_decoder_utils
            N = b200_decoder
            for name in ('block_joints', 'greedy', 'keypoint_threshold', 'keypoint_threshold_rel', 'reverse_match',
                         'force_complete', 'force_complete_caf_th'):
                getattr(N.CifCaf, 'set_' + name)(getattr(ref, 'get_' + name)())
            for name in ('neighbors', 'threshold', 'ablation_skip'):
                getattr(N.CifHr, 'set_' + name)(getattr(utl.CifHr, 'get_' + name)())
            for name in ('threshold', 'ablation_nms', 'ablation_no_rescore'):
                getattr(N.CifSeeds, 'set_' + name)(getattr(utl.CifSeeds, 'get_' + name)())
            for name in ('default_score_th', 'ablation_no_rescore'):
                getattr(N.CafScored, 'set_' + name)(getattr(utl.CafScored, 'get_' + name)())
            for name in ('suppression', 'instance_threshold', 'keypoint_threshold'):
                getattr(N.NMSKeypoints, 'set_' + name)(getattr(utl.NMSKeypoints, 'get_' + name)())

        @classmethod
        def factory(cls, head_metas):
            if openpifpaf.decoder.cifcaf.CifCafDense.dense_coupling:
                return []     # --dense-connections asks for CifCafDense (decoder/cifcaf.py:214-216)
            return [
                CifCafB200([meta], [meta_next])
                for meta, meta_next in zip(head_metas[:-1], head_metas[1:])
                if isinstance(meta, headmeta.Cif) and isinstance(meta_next, headmeta.Caf)
            ]

        def _annotations(self, ann_t, ids_t):
            """decoder/cifcaf.py:262-272"""
            out = []
            for ann_data, ann_id in zip(ann_t, ids_t):
                ann = Annotation(self.cif_metas[0].keypoints, self.caf_metas[0].skeleton,
                                 score_weights=self.score_weights)
                ann.data[:, :2] = ann_data[:, 1:3]
                ann.data[:, 2] = ann_data[:, 0]
                ann.joint_scales[:] = ann_data[:, 3]
                if ann_id != -1:
                    ann.id_ = int(ann_id)
                out.append(ann)
            return out

        def __call__(self, fields, initial_annotations=None):
            init_t = ids_t = None
            if initial_annotations:
                n = len(initial_annotations)
                init_t = torch.empty((n, self.cif_metas[0].n_fields, 4))
                ids_t = torch.empty((n,), dtype=torch.int64)
                for i, ann_py in enumerate(initial_annotations):           # decoder/cifcaf.py:228-239
                    init_t[i, :, 0] = torch.from_numpy(ann_py.data[:, 2].astype(np.float32))
                    init_t[i, :, 1] = torch.from_numpy(ann_py.data[:, 0].astype(np.float32))
                    init_t[i, :, 2] = torch.from_numpy(ann_py.data[:, 1].astype(np.float32))
                    init_t[i, :, 3] = torch.from_numpy(np.asarray(ann_py.joint_scales, dtype=np.float32))
                    ids_t[i] = getattr(ann_py, 'id_', -1)
            # the reference's C++ decoder takes the CIF field count from the tensor, not from n_keypoints: the tracking
            # pose has 2 x K keypoints over the K single-frame CIF fields (tracking_pose.py:47-65, 192-199)
            n_cif = int(fields[self.cif_metas[0].head_index].shape[0])
            if n_cif != self.native.n_cif_fields:
                self.native = b200_decoder.CifCaf(self.native.n_keypoints, self.native.skeleton, n_cif_fields=n_cif)
            self.sync_statics()
            start = time.perf_counter()
            ann_t, ids = self.native.call_with_initial_annotations(
                fields[self.cif_metas[0].head_index], self.cif_metas[0].stride,
                fields[self.caf_metas[0].head_index], self.caf_metas[0].stride, init_t, ids_t)
            LOG.debug('b200 annotations = %d (%.1fms)', len(ann_t), (time.perf_counter() - start) * 1000.0)
            return self._annotations(ann_t.numpy(), ids.numpy())

        def _compile(self, shell, h, w, batch, device_index):
            return b200_predictor.from_shell(shell, h, w, batch, device=device_index,
                                             cif_meta=self.cif_metas[0], caf_meta=self.caf_metas[0])

        def batch(self, model, image_batch, *, device=None, gt_anns_batch=None):
            """decoder/decoder.py:114-137 with everything on the GPU."""
            if not self.fast_batch or not torch.cuda.is_available():
                return super().batch(model, image_batch, device=device, gt_anns_batch=gt_anns_batch)
            self.sync_statics()
            start = time.perf_counter()
            shell = model.module if hasattr(model, 'module') else model     # DataParallel (predictor.py:33-37)
            b, _, h, w = image_batch.shape
            pred = self._predictor_for(shell, int(b), int(h), int(w), device)
            results = pred.batch(image_batch if image_batch.dtype == torch.float32 else image_batch.float())
            self.last_nn_time = self.last_decoder_time = time.perf_counter() - start
            return [self._annotations(a.numpy(), i.numpy()) for a, i in results]

    class CifCafDenseB200(Decoder):
        """decoder/cifcaf.py:17-78 (CifCafDense): the CAF and the dense CAF (caf25) heads concatenated behind one
        CifCaf decode over the concatenated skeleton.  (The dense head's decoder_confidence_scales set by the
        reference's constructor are not read by its C++ decoder, csrc/src/cifcaf.cpp:299-301 -- nor here.)"""

        def __init__(self, cif_meta, caf_meta, dense_caf_meta):
            super().__init__()
            self.cif_meta, self.caf_meta, self.dense_caf_meta = cif_meta, caf_meta, dense_caf_meta
            self.priority += 1.0 + (cif_meta.n_fields + caf_meta.n_fields + dense_caf_meta.n_fields) / 1000.0
            dense_caf_meta.decoder_confidence_scales = [
                openpifpaf.decoder.cifcaf.CifCafDense.dense_coupling for _ in dense_caf_meta.skeleton]
            concatenated = headmeta.Caf.concatenate([caf_meta, dense_caf_meta])
            self.cifcaf = CifCafB200([cif_meta], [concatenated])

        @classmethod
        def factory(cls, head_metas):
            if len(head_metas) < 3 or not openpifpaf.decoder.cifcaf.CifCafDense.dense_coupling:
                return []
            return [
                CifCafDenseB200(cif_meta, caf_meta, dense_meta)
                for cif_meta, caf_meta, dense_meta in zip(head_metas, head_metas[1:], head_metas[2:])
                if (isinstance(cif_meta, headmeta.Cif) and isinstance(caf_meta, headmeta.Caf)
                    and isinstance(dense_meta, headmeta.Caf))
            ]

        def __call__(self, fields, initial_annotations=None):
            caf = torch.cat([fields[self.caf_meta.head_index], fields[self.dense_caf_meta.head_index]], dim=0)
            cifcaf_fields = [None] * (max(self.cif_meta.head_index, self.caf_meta.head_index) + 1)
            cifcaf_fields[self.cif_meta.head_index] = fields[self.cif_meta.head_index]
            cifcaf_fields[self.caf_meta.head_index] = caf
            return self.cifcaf(cifcaf_fields, initial_annotations=initial_annotations)

    class CifDetB200(_CompileCache, Decoder):
        """decoder/cifdet.py:15-96 with the C++ CifDet call AND the torchvision NMS / score filter on the GPU
        (libpifpaf_b200 pifpaf_cifdet_*).  Class attributes are read from the reference's CifDet at call time, so
        decoder.factory.configure (decoder/factory.py:68,78) keeps configuring one source of truth."""
        fast_batch = True

        def __init__(self, head_metas):
            super().__init__()
            self.metas = head_metas
            self.priority = -1.0 + 0.5                      # decoder/cifdet.py:29 is -1.0: outrank it, stay below poses
            self.priority += sum(m.n_fields for m in head_metas) / 1000.0
            self.native = b200_decoder.CifDet(head_metas[0].n_fields)
            self._compiled = collections.OrderedDict()

        @classmethod
        def configure(cls, args):
            """The flags CifCafB200.cli owns (--b200-no-fast-batch, --b200-compile-cache) apply here too."""
            cls.fast_batch = getattr(args, 'b200_fast_batch', True)
            cls.compile_cache_size = max(1, int(getattr(args, 'b200_compile_cache', cls.compile_cache_size)))

        @classmethod
        def factory(cls, head_metas):
            return [CifDetB200([meta]) for meta in head_metas if isinstance(meta, headmeta.CifDet)]

        @staticmethod
        def sync_statics():
            utl = torch.classes.openpifpaf_decoder_utils
            b200_decoder.CifHr.set_neighbors(utl.CifHr.get_neighbors())
            b200_decoder.CifHr.set_threshold(utl.CifHr.get_threshold())
            b200_decoder.CifDetSeeds.set_threshold(utl.CifDetSeeds.get_threshold())
            b200_decoder.CifDet.set_max_detections_before_nms(
                torch.classes.openpifpaf_decoder.CifDet.get_max_detections_before_nms())

        @staticmethod
        def nms_params():
            """the NMS and score filter of the reference's CifDet wrapper (decoder/cifdet.py:55-64), by value"""
            ref = openpifpaf.decoder.CifDet
            return dict(iou_threshold=ref.iou_threshold, nms_by_category=ref.nms_by_category,
                        suppression=ref.suppression, instance_threshold=ref.instance_threshold)

        def __call__(self, fields):
            self.sync_statics()
            field = fields[self.metas[0].head_index]
            if not field.is_cuda:
                field = field.cuda(self.native.device)
            return self._annotations(*self.native.decode_batch(
                field[:, :6].unsqueeze(0), self.metas[0].stride, nms=True, **self.nms_params())[0])

        def _compile(self, shell, h, w, batch, device_index):
            if len(shell.head_metas) != 1:
                raise b200_network.UnsupportedModel('the GPU detection path compiles Shells with one CifDet head')
            return b200_predictor.from_shell(shell, h, w, batch, device=device_index)

        def batch(self, model, image_batch, *, device=None, gt_anns_batch=None):
            """decoder/decoder.py:114-137 with the forward, the decode and the NMS on the GPU.  A model the compiled
            forward does not implement takes the reference's Decoder.batch (stock forward, then __call__ per image)."""
            if not self.fast_batch or not torch.cuda.is_available():
                return super().batch(model, image_batch, device=device, gt_anns_batch=gt_anns_batch)
            start = time.perf_counter()
            shell = model.module if hasattr(model, 'module') else model     # DataParallel (predictor.py:33-37)
            b, _, h, w = image_batch.shape
            try:
                pred = self._predictor_for(shell, int(b), int(h), int(w), device)
            except b200_network.UnsupportedModel as e:
                LOG.info('CifDetB200: %s; decoding through the reference batch path', e)
                return super().batch(model, image_batch, device=device, gt_anns_batch=gt_anns_batch)
            self.sync_statics()
            pred.nms_params = self.nms_params()
            results = pred.batch(image_batch if image_batch.dtype == torch.float32 else image_batch.float())
            self.last_nn_time = self.last_decoder_time = time.perf_counter() - start
            return [self._annotations(*r) for r in results]

        def _annotations(self, cats, scores, boxes):
            from openpifpaf.annotation import AnnotationDet
            boxes_np = boxes.numpy()
            boxes_np[:, 2:] -= boxes_np[:, :2]              # xyxy -> xywh (decoder/cifdet.py:86-87)
            out = []
            for category, score, box in zip(cats, scores, boxes_np):
                ann = AnnotationDet(self.metas[0].categories)
                ann.set(int(category), float(score), box)
                out.append(ann)
            return out

    class TrackingPoseB200(openpifpaf.decoder.TrackingPose):
        """decoder/tracking_pose.py:18-296 (TrackingPose): the tracker's Python bookkeeping (active tracks, soft NMS over
        tracks, track recovery, pruning) is the reference's own, inherited unchanged; what runs per frame on the hot
        path -- the CifCaf decode of the 2 x K-keypoint "tracking pose" over [cif, cat(caf, tcaf)] seeded with the
        previous frame's poses (``call_with_initial_annotations``, csrc/src/cifcaf.cpp:177-202; tracking_pose.py:165-218)
        -- goes to the GPU decoder: the reference constructor takes a ``pose_generator`` and this class hands it a
        CifCafB200 over the tracking metas."""

        def __init__(self, cif_meta, caf_meta, tcaf_meta):
            super().__init__(cif_meta, caf_meta, tcaf_meta)
            self.pose_generator = CifCafB200([self.tracking_cif_meta], [self.tracking_caf_meta])
            self.priority += 1.0          # outrank the reference's TrackingPose (tracking_pose.py:36-39: same base)

        @classmethod
        def cli(cls, parser):
            """The reference's TrackingPose.cli already owns --trackingpose-* (both classes sit in DECODERS)."""

        @classmethod
        def configure(cls, args):
            cls.track_recovery = args.trackingpose_track_recovery
            cls.single_seed = args.trackingpose_single_seed

    return openpifpaf, CifCafB200, CifCafDenseB200, CifDetB200, TrackingPoseB200


_CLASS = None


def decoder_class():
    global _CLASS
    if _CLASS is None:
        _CLASS = _build_class()[1]
    return _CLASS


def register():
    openpifpaf, cls, dense_cls, det_cls, track_cls = _build_class()
    global _CLASS
    _CLASS = cls
    openpifpaf.DECODERS.add(cls)
    openpifpaf.DECODERS.add(dense_cls)
    openpifpaf.DECODERS.add(det_cls)
    openpifpaf.DECODERS.add(track_cls)

    # Predictor calls Multi.batch (predictor.py:131); let it delegate to the GPU-resident batch path when the
    # selected decoder provides one.
    Multi = openpifpaf.decoder.multi.Multi
    if not getattr(Multi, '_b200_patched', False):
        original = Multi.batch

        def batch(self, model, image_batch, *, device=None, gt_anns_batch=None):
            decs = [d for d in self.decoders if d is not None]
            if len(decs) == 1 and isinstance(decs[0], (cls, det_cls)) and type(decs[0]).fast_batch:
                res = decs[0].batch(model, image_batch, device=device, gt_anns_batch=gt_anns_batch)
                self.last_nn_time, self.last_decoder_time = decs[0].last_nn_time, 0.0
                return res
            return original(self, model, image_batch, device=device, gt_anns_batch=gt_anns_batch)

        Multi.batch = batch
        Multi._b200_patched = True
