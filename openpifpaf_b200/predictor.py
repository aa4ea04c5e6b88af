import os
"""End-to-end batch API: images -> backbone+heads -> CifCaf decode -> annotations.

Mirror of the reference's hot loop (paths relative to the reference's src/openpifpaf/):
  Predictor.enumerated_dataloader   predictor.py:118-153
  Decoder.batch / fields_batch      decoder/decoder.py:76-137

Differences by design: the head tensors never leave the GPU (the reference does
``heads.cpu()`` at decoder/decoder.py:98 and decodes on host cores); the whole
batch is decoded by one batched launch sequence; only the final annotations
(a few KB) are copied back.  With ``overlap_decode`` the decode of batch i runs
on its own stream (on SMs the forward's persistent grids leave free) under the
forward of batch i+1; the head outputs are double buffered for that.
"""
import math
import time

import numpy as np
import torch

from . import decoder as _decoder
from . import network as _network
from . import preprocess as _preprocess


def raw_image_chunks(images, max_batch, fill):
    """Split the images of `Predictor.raw_images` into batches of at most max_batch; yields (images, fill) per batch.
    A per-image fill list (`preprocess.pad_fills`) must have one entry per image and is sliced with the images; any
    other fill applies to every batch as it is."""
    if isinstance(fill, list) and len(fill) != len(images):
        raise RuntimeError(f'fill has {len(fill)} colours for {len(images)} images')
    for i in range(0, len(images), max_batch):
        yield images[i:i + max_batch], fill[i:i + max_batch] if isinstance(fill, list) else fill


def tight_pad_groups(sizes, long_edge, max_batch, capacity, multiple=16):
    """The batches of `Predictor.raw_images(tight_pad=True)`: images (w, h) go through RescaleAbsolute(long_edge) (none
    when long_edge is None) and CenterPadTight(multiple) (transforms/pad.py:62-110), whose canvas depends on the aspect
    ratio.  Returns [((canvas_h, canvas_w), [image indices])] in order of each canvas's first image, every list in input
    order and at most max_batch long.  A canvas above capacity (h, w) raises RuntimeError."""
    groups = {}
    for i, (w, h) in enumerate(sizes):
        tw, th = _preprocess.rescale_target(w, h, long_edge) if long_edge else (w, h)
        canvas = (math.ceil((th - 1) / multiple) * multiple + 1, math.ceil((tw - 1) / multiple) * multiple + 1)
        if canvas[0] > capacity[0] or canvas[1] > capacity[1]:
            raise RuntimeError(f'image {i} ({w}x{h}) pads to a {canvas[1]}x{canvas[0]} canvas, above the net\'s '
                               f'{capacity[1]}x{capacity[0]}')
        groups.setdefault(canvas, []).append(i)
    return [(canvas, idx[k:k + max_batch]) for canvas, idx in groups.items() for k in range(0, len(idx), max_batch)]


class Predictor:
    """:param net: `network.CompiledNet`
    :param n_keypoints: number of keypoints of the CIF head
    :param skeleton: 1-based skeleton of the CAF head (``headmeta.Caf.skeleton``)
    :param cif_head, caf_head: indices of the two heads in the model output (``headmeta.head_index``)
    :param overlap_decode: decode on a second stream, concurrently with the next forward
    :param reserve_sms: SMs kept free of the forward's persistent grids for the concurrent decode
                        (None: one per image of the batch, at most 1/8 of the GPU)"""

    def __init__(self, net, n_keypoints, skeleton, *, device=0, cif_head=0, caf_head=1,
                 overlap_decode=False, reserve_sms=None):
        sk = torch.as_tensor(skeleton, dtype=torch.int64).reshape(-1, 2) - 1     # decoder/cifcaf.py:121
        self.decoder = _decoder.CifCaf(n_keypoints, sk, device=device)
        # size the native handle once, from the net (never re-created while results are in flight)
        hd = net.heads[cif_head]
        self.decoder.reserve(net.max_batch, hd['h'], hd['w'], max(net.heads[cif_head]['stride'], net.heads[caf_head]['stride']))
        self.cif_head, self.caf_head = int(cif_head), int(caf_head)
        self._setup(net, device, overlap_decode, reserve_sms)

    def _setup(self, net, device, overlap_decode, reserve_sms):
        """What every predictor has besides its decoder: the net, the streams, the overlap policy."""
        self.net = net
        self.device = torch.device('cuda', device)
        self.stream = torch.cuda.Stream(device=self.device)
        self.copy_stream = torch.cuda.Stream(device=self.device)
        self.dec_stream = torch.cuda.Stream(device=self.device)
        self.overlap_decode = bool(overlap_decode)
        self._dec_done = [None, None]
        self._step = 0
        if self.overlap_decode:
            net.set_head_buffers(2)
            n_sm = torch.cuda.get_device_properties(self.device).multi_processor_count
            if reserve_sms is None:
                env = os.environ.get('PIFPAF_RESERVE_SMS')
                # at 64 images per step the network wants every SM, at 8-16 images the decode wants 8 of its own
                reserve_sms = int(env) if env is not None else (8 if net.max_batch <= 16 else 4 if net.max_batch <= 32 else 0)
            net.set_sm_limit(n_sm - int(reserve_sms) if reserve_sms else 0)
        self._dev_images = None
        self.last_nn_time = 0.0
        self.last_decoder_time = 0.0
        self.image_mean = _network.CompiledNet.IMAGE_MEAN
        self.image_std = _network.CompiledNet.IMAGE_STD
        #: benchmark hook: (cif [B,F,5,h,w], cif_stride, caf [B,C,8,h,w], caf_stride) CUDA tensors decoded INSTEAD of
        #: the network's own head outputs (random-init weights emit no poses; planted fields give the decoder the
        #: work of real images).  None in production.
        self.decode_fields_override = None

    def close(self):
        """Free the GPU buffers of the compiled net and the decoder workspace now (not at garbage collection)."""
        torch.cuda.synchronize(self.device)
        self.decoder._free()
        self.net.close()
        if getattr(self, '_jpeg', None) is not None:
            self._jpeg.close()
            self._jpeg = None

    def fields_batch(self, image_batch):
        """decoder/decoder.py:76-112 without the .cpu(): returns device-resident head tensors."""
        return self._forward(image_batch)

    def _forward(self, image_batch_dev):
        """float32 [B,3,H,W] (already normalised, what the reference's dataloader yields) or raw uint8 [B,H,W,3]
        (ToTensor + Normalize of transforms/__init__.py:26-33 fused into the stem kernel)."""
        if image_batch_dev.dtype == torch.uint8:
            return self.net.forward_uint8(image_batch_dev, mean=self.image_mean, std=self.image_std)
        return self.net.forward(image_batch_dev)

    def _decode_inputs(self, heads, batch):
        if self.decode_fields_override is not None:
            cif, cs, caf, fs = self.decode_fields_override
            return cif[:batch], cs, caf[:batch], fs
        return (heads[self.cif_head], self.net.heads[self.cif_head]['stride'],
                heads[self.caf_head], self.net.heads[self.caf_head]['stride'])

    def _decode_async(self, heads, batch, stream=None):
        cif, cs, caf, fs = self._decode_inputs(heads, batch)
        self.decoder.decode_batch_async(cif, cs, caf, fs, stream=stream)

    def batch_device(self, image_batch_dev):
        """Device-resident images -> enqueue forward + decode (no host sync).  The forward goes to the current
        stream; the decode to the current stream too, or, with overlap_decode, to the decode stream behind an event
        (call join() before timing or reusing the current stream's results)."""
        cur = torch.cuda.current_stream(self.device)
        if not self.overlap_decode:
            heads = self._forward(image_batch_dev)
            self._decode_async(heads, int(image_batch_dev.shape[0]))
            return
        slot = self._step & 1
        self._step += 1
        if self._dec_done[slot] is not None:
            cur.wait_event(self._dec_done[slot])       # the head-output set this forward overwrites has been decoded
        heads = self._forward(image_batch_dev)
        ready = torch.cuda.Event()
        ready.record(cur)
        self.dec_stream.wait_event(ready)
        self._decode_async(heads, int(image_batch_dev.shape[0]), stream=self.dec_stream)
        done = torch.cuda.Event()
        done.record(self.dec_stream)
        self._dec_done[slot] = done

    def result_stream(self):
        """The stream the decode results are produced on."""
        return self.dec_stream if self.overlap_decode else torch.cuda.current_stream(self.device)

    def join(self):
        """Make the current stream wait for every decode enqueued so far (overlap_decode)."""
        cur = torch.cuda.current_stream(self.device)
        for ev in self._dec_done:
            if ev is not None:
                cur.wait_event(ev)

    def batch(self, image_batch_host):
        """decoder/decoder.py:114-137: image batch (host, ideally pinned; float32 [B,3,H,W] normalised, or raw
        uint8 [B,H,W,3]) -> per-image (annotations [N,K,4], ids [N]) CPU tensors.  H2D, forward, decode and D2H
        all inside."""
        t0 = time.perf_counter()
        with torch.cuda.stream(self.stream):
            if (self._dev_images is None or self._dev_images.shape != image_batch_host.shape
                    or self._dev_images.dtype != image_batch_host.dtype):
                self._dev_images = torch.empty(image_batch_host.shape, dtype=image_batch_host.dtype, device=self.device)
            self._dev_images.copy_(image_batch_host, non_blocking=True)
            self.batch_device(self._dev_images)
            result = self.decoder.fetch(stream=self.result_stream())
            self.join()
        self.last_nn_time = self.last_decoder_time = time.perf_counter() - t0
        return result

    def raw_images(self, images, *, json_data=False, fill=None, score_weights=None, fast_rescaling=True,
                   opencv_rescaling=False, tight_pad=False, long_edge=None):
        """The reference's Predictor.numpy_images / images (predictor.py:155-196) for a list of RAW uint8 [h, w, 3]
        images with everything after the JPEG decode on the GPU: RescaleAbsolute(long edge = the compiled input size)
        + CenterPad (`preprocess.GpuPreprocess`, bit-identical to the reference's Pillow path), ToTensor + Normalize in
        the stem, forward, decode; then `Annotation.inverse_transform` (and `json_data`) for all annotations of an
        image at once.  fill: the pad colour as for `GpuPreprocess` (a list has one colour per image of `images`).
        fast_rescaling: the reference's Predictor.fast_rescaling; False (its --precise-rescaling) rescales like
        scipy.ndimage.zoom(order=1) instead of Pillow (`GpuPreprocess(fast_rescaling=False)`).
        opencv_rescaling: True rescales like cv2.resize(INTER_LINEAR), which the reference's fast rescale uses when
        OpenCV is importable (`GpuPreprocess(opencv=True)`); with fast_rescaling=False scipy is used either way, as in
        the reference.
        tight_pad: pad like the reference's Predictor at batch size 1 instead: RescaleAbsolute(long_edge) (no rescale
        with long_edge None, the reference's default) + CenterPadTight(16), the pad colour (124, 116, 104) unless `fill`
        says otherwise.  Images are grouped by canvas into batches of at most max_batch, each group runs at its canvas
        size on this one net (`CompiledNet.set_input_size`) and is decoded at its field size; a canvas larger than the
        net's input raises RuntimeError before anything is enqueued.
        Returns per image, in input order, (data [N, K, 3] (x, y, v) in original-image pixels, joint_scales [N, K],
        meta) or, with json_data, (list of dicts, meta)."""
        if tight_pad:
            return self._tight_pad_images(images, json_data, fill, score_weights, fast_rescaling, opencv_rescaling,
                                          long_edge)
        if long_edge is not None:
            raise RuntimeError('long_edge applies to tight_pad=True; the square canvas is the net\'s input size')
        if self.net.in_h != self.net.in_w:
            raise RuntimeError('raw_images needs a net compiled for a square input (CenterPad(long_edge))')
        if getattr(self, '_gpu_preprocess', None) is None:
            self._gpu_preprocess = {}
        key = (bool(fast_rescaling), bool(fast_rescaling) and bool(opencv_rescaling))
        if key not in self._gpu_preprocess:
            self._gpu_preprocess[key] = _preprocess.GpuPreprocess(
                self.net.in_w, batched=True, fast_rescaling=key[0], opencv=key[1], device=self.device.index)
        preprocess = self._gpu_preprocess[key]
        out = []
        for chunk, chunk_fill in raw_image_chunks(images, self.net.max_batch, fill):
            with torch.cuda.stream(self.stream):
                canvas, metas = preprocess(chunk, fill=chunk_fill, stream=self.stream)
                self.batch_device(canvas)
                result = self.decoder.fetch(stream=self.result_stream())
                self.join()
            out += [self._result(ann, meta, json_data, score_weights) for (ann, _), meta in zip(result, metas)]
        return out

    @staticmethod
    def _result(ann, meta, json_data, score_weights):
        data, scales = _preprocess.inverse_transform_batch(ann.numpy(), meta)
        if json_data:
            return _preprocess.json_data_batch(data, scales, score_weights=score_weights), meta
        return data, scales, meta

    def _tight_pad_images(self, images, json_data, fill, score_weights, fast_rescaling, opencv_rescaling, long_edge):
        """raw_images(tight_pad=True): one GpuPreprocess(batched=False) call, forward and decode per canvas group; the
        net's input size is restored afterwards"""
        sizes = []
        for im in images:
            if im.dtype not in (np.uint8, torch.uint8) or len(im.shape) != 3 or im.shape[2] != 3:
                raise RuntimeError('images must be uint8 [h, w, 3]')
            sizes.append((int(im.shape[1]), int(im.shape[0])))
        groups = tight_pad_groups(sizes, long_edge, self.net.max_batch, (self.net.in_h, self.net.in_w))
        fills = _preprocess.pad_fills(fill, len(images), False)
        key = ('tight', long_edge, bool(fast_rescaling), bool(fast_rescaling) and bool(opencv_rescaling))
        if getattr(self, '_gpu_preprocess', None) is None:
            self._gpu_preprocess = {}
        if key not in self._gpu_preprocess:
            self._gpu_preprocess[key] = _preprocess.GpuPreprocess(long_edge, batched=False, fast_rescaling=key[2],
                                                                  opencv=key[3], device=self.device.index)
        preprocess = self._gpu_preprocess[key]
        out = [None] * len(images)
        restore = self.net.input_size
        try:
            for canvas_hw, idx in groups:
                self.net.set_input_size(*canvas_hw)
                with torch.cuda.stream(self.stream):
                    canvas, metas = preprocess([images[i] for i in idx], fill=[fills[i] for i in idx],
                                               stream=self.stream)
                    self.batch_device(canvas)
                    result = self.decoder.fetch(stream=self.result_stream())
                    self.join()
                for i, (ann, _), meta in zip(idx, result, metas):
                    out[i] = self._result(ann, meta, json_data, score_weights)
        finally:
            self.net.set_input_size(*restore)
        return out

    def jpeg_images(self, files_or_bytes, *, json_data=False, fill=None, score_weights=None, fast_rescaling=True,
                    opencv_rescaling=False, tight_pad=False, long_edge=None):
        """`raw_images` of the JPEG files (paths or bytes) decoded like the reference's Predictor.images
        (PIL.Image.open(f).convert('RGB'), datasets/image_list.py:18), but on the GPU (`preprocess.GpuJpegDecoder`;
        streams it does not decode are decoded by Pillow).  Chunked by max_batch; each chunk's decode is enqueued on
        the predictor's stream ahead of its resize (fast_rescaling, opencv_rescaling, tight_pad and long_edge as for
        raw_images).  Returns what raw_images returns, per file."""
        files = list(files_or_bytes)
        if isinstance(fill, list) and len(fill) != len(files):
            raise RuntimeError(f'fill has {len(fill)} colours for {len(files)} images')
        out = []
        for chunk, chunk_fill in raw_image_chunks(files, self.net.max_batch, fill):
            datas = [_preprocess.read_stream(f) for f in chunk]
            dec = self._jpeg_decoder(datas)
            images, _ = dec(datas, stream=self.stream, host_pillow=True)
            out.extend(self.raw_images(images, json_data=json_data, fill=chunk_fill, score_weights=score_weights,
                                       fast_rescaling=fast_rescaling, opencv_rescaling=opencv_rescaling,
                                       tight_pad=tight_pad, long_edge=long_edge))
        return out

    def _jpeg_decoder(self, datas):
        """the JPEG decoder, sized from the chunk's frame headers; re-created (after the work in flight) when a chunk
        does not fit, at the larger of the old capacities and the chunk's needs"""
        fp = [_preprocess.jpeg_footprint(d) for d in datas]
        need = (len(datas), sum(len(d) for d in datas), max(p for p, _ in fp), sum(b for _, b in fp),
                sum(p for p, _ in fp))
        dec = getattr(self, '_jpeg', None)
        if dec is None or not dec.fits(*need):
            old = (0, 0, 0, 0)
            if dec is not None:
                torch.cuda.synchronize(self.device)
                dec.close()
                old = (dec.max_bytes, dec.max_pixels, dec.max_blocks, dec.out_pixels)
            self._jpeg = _preprocess.GpuJpegDecoder(
                self.net.max_batch, max(need[1], old[0]), max(need[2], old[1], 1), max_blocks=max(need[3], old[2], 1),
                out_pixels=max(need[4], old[3], 1), device=self.device.index)
        return self._jpeg

    def batches(self, host_batches):
        """Pipelined variant of `batch` over an iterable of host image batches (what Predictor.dataloader /
        enumerated_dataloader does in the reference, predictor.py:118-153): the H2D copy of batch i+1 runs on a
        copy stream under the forward+decode of batch i, and the (tiny) result D2H of batch i is waited for
        only after batch i+1 has been enqueued.  Yields per-batch results in order."""
        dev, copied, consumed = [None, None], [None, None], [None, None]
        outstanding = 0
        for i, host in enumerate(host_batches):
            s = i % 2
            if dev[s] is None or dev[s].shape != host.shape or dev[s].dtype != host.dtype:
                dev[s] = torch.empty(host.shape, dtype=host.dtype, device=self.device)
                copied[s], consumed[s] = torch.cuda.Event(), None
            with torch.cuda.stream(self.copy_stream):
                if consumed[s] is not None:
                    self.copy_stream.wait_event(consumed[s])
                dev[s].copy_(host, non_blocking=True)
                copied[s].record(self.copy_stream)
            with torch.cuda.stream(self.stream):
                self.stream.wait_event(copied[s])
                self.batch_device(dev[s])
                consumed[s] = torch.cuda.Event()
                consumed[s].record(self.stream)        # the forward (the only reader of dev[s]) is on self.stream
                self.decoder.fetch_begin(stream=self.result_stream())
            outstanding += 1
            if outstanding == 2:
                yield self.decoder.fetch_end()
                outstanding -= 1
        while outstanding:
            yield self.decoder.fetch_end()
            outstanding -= 1
        with torch.cuda.stream(self.stream):
            self.join()


class DetPredictor(Predictor):
    """Predictor of a detection Shell (one CifDet head, headmeta.py:117-125): `batch`, `batch_device` + `fetch`
    and `fields_batch` as for poses; per image the result is (categories [N] int64 (1-based), scores [N], boxes [N, 4]
    (x1, y1, x2, y2)) of `decoder.CifDet.decode_batch(nms=True)`, with the NMS and score filter of the reference's
    CifDet wrapper (decoder/cifdet.py:55-64).  Those four parameters (`nms_params`) go by value into every decode.
    Overlapped decode, `batches()` and `raw_images()` are not implemented for detection."""

    def __init__(self, net, n_categories, *, device=0, head=0, iou_threshold=0.5, nms_by_category=True,
                 suppression=0.1, instance_threshold=0.15, overlap_decode=False):
        if overlap_decode:
            raise RuntimeError('overlap_decode is not implemented for detection (it needs a double-buffered CifDet '
                               'fetch)')
        self.decoder = _decoder.CifDet(n_categories, device=device)
        self.head = int(head)
        self.nms_params = dict(iou_threshold=iou_threshold, nms_by_category=nms_by_category, suppression=suppression,
                               instance_threshold=instance_threshold)
        self._setup(net, device, False, None)

    def _decode_async(self, heads, batch, stream=None):
        self.decoder.decode_batch_async(heads[self.head][:batch], self.net.heads[self.head]['stride'], nms=True,
                                        stream=stream, **self.nms_params)

    def batches(self, host_batches):
        raise RuntimeError('batches() is not implemented for detection (it needs a double-buffered CifDet fetch); '
                           'call batch() per batch')

    def raw_images(self, images, **kwargs):
        raise RuntimeError('raw_images() is not implemented for detection (no inverse transform of boxes); '
                           'preprocess on the host and call batch()')

    def jpeg_images(self, files_or_bytes, **kwargs):
        raise RuntimeError('jpeg_images() is not implemented for detection (no inverse transform of boxes); '
                           'preprocess on the host and call batch()')


def is_cifdet_meta(meta):
    """headmeta.CifDet by its component layout: one confidence, two vectors (offset, no offset), no scale."""
    return ((int(meta.n_confidences), int(meta.n_vectors), int(meta.n_scales), tuple(meta.vector_offsets))
            == (1, 2, 0, (True, False)))


def from_shell(shell, in_h, in_w, max_batch, *, device=0, cif_meta=None, caf_meta=None, **kwargs):
    """Compile a reference-style Shell (network/nets.py:7-48) with a (Cif, Caf) head pair into a Predictor, or a
    Shell whose only head is a CifDet into a DetPredictor (kwargs: its NMS parameters).
    cif_meta / caf_meta: the head metas the decoder was built for (decoder/cifcaf.py:212-222); default: the
    first Cif-like meta followed by a Caf-like one."""
    plan = _network.plan_from_shell(shell)
    net = _network.CompiledNet(plan, in_h, in_w, max_batch, device=device)
    metas = list(shell.head_metas)
    if len(metas) == 1 and is_cifdet_meta(metas[0]):
        return DetPredictor(net, metas[0].n_fields, device=device, **kwargs)
    if cif_meta is None or caf_meta is None:
        cif_meta, caf_meta = metas[0], metas[1]
    skeleton = getattr(caf_meta, 'skeleton', None)
    if skeleton is None:
        raise RuntimeError('CAF head meta has no skeleton')

    def index_of(meta, default):
        hi = getattr(meta, 'head_index', None)
        return int(hi) if hi is not None else default

    return Predictor(net, cif_meta.n_fields, skeleton, device=device,
                     cif_head=index_of(cif_meta, 0), caf_head=index_of(caf_meta, 1), **kwargs)
