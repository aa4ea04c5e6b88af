"""GPU: detection models end to end -- `predictor.from_shell` on a Shell with one CifDet head (the resnet18-cocodet
recipe: second input conv, dilated block5, 91 categories, upsample-2 head) gives a DetPredictor whose batch /
batch_device / fields_batch results equal `decoder.CifDet.decode_batch(nms=True)` on the compiled net's own fields;
the split decode (decode_batch_async + fetch) equals decode_batch; the paths detection does not implement refuse
loudly."""
import numpy as np
import pytest
import torch

import det_models
from openpifpaf_b200 import decoder, network, predictor

pytestmark = pytest.mark.gpu


def assert_same(got, want):
    assert len(got) == len(want)
    for (c, s, b), (wc, ws, wb) in zip(got, want):
        assert torch.equal(c, wc) and torch.equal(s, ws) and torch.equal(b, wb)


@pytest.fixture(scope='module')
def det():
    shell = det_models.calibrate_det_head(det_models.make_variant_shell('cocodet', seed=0))
    pred = predictor.from_shell(shell, 161, 161, 4)
    images = torch.randn(4, 3, 161, 161, generator=torch.Generator().manual_seed(3)).pin_memory()
    return shell, pred, images


def test_from_shell_builds_a_det_predictor(det):
    shell, pred, _ = det
    assert isinstance(pred, predictor.DetPredictor)
    assert pred.net.heads[0]['stride'] == shell.head_nets[0].meta.stride == 8
    assert (pred.net.heads[0]['n_fields'], pred.net.heads[0]['n_comp']) == (91, 6)


def test_batch_equals_decode_batch_on_the_nets_fields(det):
    _, pred, images = det
    for b in (4, 2):           # a smaller batch reuses the net and the decoder workspace
        res = pred.batch(images[:b])
        assert len(res) == b
        counts = [len(c) for c, _, _ in res]
        assert all(n > 0 for n in counts), counts
        (field,) = pred.fields_batch(images[:b].cuda())
        assert tuple(field.shape) == (b, 91, 6, 21, 21)
        want = decoder.CifDet(91).decode_batch(field, 8, nms=True)
        assert_same(res, want)
        # the same through batch_device + fetch on the current stream
        pred.batch_device(images[:b].cuda())
        assert_same(pred.decoder.fetch(), want)
        for c, s, bx in res:
            assert c.dtype == torch.int64 and (c >= 1).all() and (c <= 91).all()
            assert (s > 0.15).all() and (bx[:, 2:] >= bx[:, :2]).all()


def test_nms_parameters_go_by_value(det):
    _, pred, images = det
    base = sum(len(c) for c, _, _ in pred.batch(images))
    pred.nms_params = dict(pred.nms_params, instance_threshold=0.9)
    try:
        strict = sum(len(c) for c, _, _ in pred.batch(images))
    finally:
        pred.nms_params = dict(pred.nms_params, instance_threshold=0.15)
    assert strict < base


def test_split_decode_equals_decode_batch(det):
    _, pred, images = det
    (field,) = pred.fields_batch(images.cuda())
    field = field.clone()
    dec = decoder.CifDet(91)
    for nms in (False, True):
        want = dec.decode_batch(field, 8, nms=nms)
        dec.decode_batch_async(field, 8, nms=nms)
        assert_same(dec.fetch(), want)
    with pytest.raises(RuntimeError, match='decode_batch_async'):
        dec.fetch()


def test_unimplemented_detection_paths_refuse(det):
    _, pred, images = det
    with pytest.raises(RuntimeError, match='detection'):
        list(pred.batches([images]))
    with pytest.raises(RuntimeError, match='detection'):
        pred.raw_images([np.zeros((161, 161, 3), dtype=np.uint8)])
    with pytest.raises(RuntimeError, match='overlap_decode'):
        predictor.DetPredictor(pred.net, 91, overlap_decode=True)


def test_refused_model_raises_unsupported_model():
    base = det_models.make_resnet('resnet18', remove_last_block=True)
    with pytest.raises(network.UnsupportedModel):
        predictor.from_shell(det_models.make_det_shell(base, 3, 1), 97, 97, 1)
