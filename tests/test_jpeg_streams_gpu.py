"""GPU: pifpaf_jpeg_decode on the streams of tests/jpeg_streams.py -- damaged scans, restart markers missing, repeated
or renumbered, trailers, table placement, colour-space signalling and re-encoded scans -- interleaved with clean
streams, under every round cap: each image equals Pillow's byte for byte and the round / fallback counters equal the
restatement's.  Streams Pillow refuses raise without writing, and the handle decodes the next batch.  A trailer is
neither staged nor counted against max_bytes."""
import io

import numpy as np
import pytest
import torch

from openpifpaf_b200 import preprocess as pp
import jpeg_ref as jr
import jpeg_streams as js
from test_jpeg import CORPUS, encode
from test_jpeg_gpu import assert_equal_pillow, expected_stats

PIL = pytest.importorskip('PIL.Image')


def pillow_decodes(data):
    try:
        PIL.open(io.BytesIO(data)).convert('RGB')
        return True
    except OSError:
        return False


def split_corpus():
    """(GPU-route streams Pillow decodes, streams Pillow refuses)"""
    gpu, refused = [], []
    for name, d in sorted(js.corpus().items()):
        if not pillow_decodes(d):
            refused.append(d)
        elif jr.parse(d)[0] == 'gpu':
            gpu.append(d)
    return gpu, refused


@pytest.mark.gpu
def test_corpus_streams_in_mixed_batches_equal_pillow():
    gpu, _ = split_corpus()
    assert len(gpu) == 125                           # every GPU-route stream of the corpus (test_routes_of_the_corpus)
    clean = [encode(h, w, seed=i, **opts) for i, (h, w, opts) in enumerate(CORPUS[:12])]
    batch = []
    for i, d in enumerate(gpu):                      # a clean stream after every fourth corpus stream
        batch.append(d)
        if i % 4 == 3:
            batch.append(clean[(i // 4) % len(clean)])
    halves = [batch[:len(batch) // 2], batch[len(batch) // 2:]]
    n_img = max(len(h) for h in halves)
    dec = pp.GpuJpegDecoder(n_img, 2 * max(sum(len(d) for d in h) for h in halves) + (1 << 16), 401 * 400)
    for datas in halves:
        for cap in (-1, 0, 1, 2):
            images, routes = dec(datas, max_rounds=cap)
            assert routes == ['gpu'] * len(datas)
            torch.cuda.synchronize()
            assert_equal_pillow(images, datas)
            st = dec.stats()
            assert (st['sync_rounds'], st['fallbacks']) == expected_stats(datas, cap), (cap, st)
    dec.close()


@pytest.mark.gpu
def test_pillow_refused_streams_raise_write_nothing_and_the_handle_recovers():
    gpu, refused = split_corpus()
    assert refused
    dec = pp.GpuJpegDecoder(8, 1 << 16, 64 * 64)
    dec._out.fill_(7)
    torch.cuda.synchronize()
    for bad in refused:
        with pytest.raises(OSError):                 # routed to Pillow, which refuses it as the reference's loader would
            dec([bad])
        torch.cuda.synchronize()
        assert bool((dec._out == 7).all())
    good = gpu[:8]
    images, routes = dec(good)
    assert routes == ['gpu'] * len(good)
    assert_equal_pillow(images, good)
    dec.close()


@pytest.mark.gpu
def test_large_photo_with_a_trailer_fits_a_handle_sized_to_its_scan():
    """a 4032 x 3024 photo followed by 3 MB of trailer (a phone's motion-photo video, with marker bytes in it): the
    scan alone is staged"""
    photo = encode(3024, 4032, seed=11, quality=92, subsampling=2)
    trailer = bytearray(js.random_bytes(31, 3 << 20))
    trailer[1000:1002] = b'\xff\xd9'
    trailer[5000:5002] = b'\xff\xd0'
    data = photo + bytes(trailer)
    route, hdr = jr.parse(data)
    assert route == 'gpu' and hdr['seg'] == jr.parse(photo)[1]['seg']
    dec = pp.GpuJpegDecoder(1, hdr['seg'][1] - hdr['seg'][0], 4032 * 3024)
    images, routes = dec([data])
    assert routes == ['gpu']
    assert_equal_pillow(images, [data])
    with pytest.raises(RuntimeError, match='max_bytes'):
        dec([photo[:-2] + b'\x00' + photo[-2:]])     # one scan byte more
    dec.close()
