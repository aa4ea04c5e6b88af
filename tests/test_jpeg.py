"""CPU: the Python restatement of the GPU JPEG decoder (tests/jpeg_ref.py) equals Pillow bit for bit on a seeded
corpus Pillow encodes here; the self-synchronising Huffman decode equals the serial one under every subsequence size
and round cap; streams the GPU does not decode are routed to Pillow and malformed streams are refused."""
import io

import numpy as np
import pytest

import jpeg_ref as jr
from openpifpaf_b200 import synth

PIL = pytest.importorskip('PIL.Image')

# (h, w, options): sizes of 1 pixel, 1 x N, N x 1, no MCU multiple, up to ~400 px; every subsampling, qualities 1 to
# 100, optimized tables, restart markers every few blocks or rows, grayscale
CORPUS = [
    (1, 1, dict(quality=75, subsampling=2)), (1, 1, dict(quality=75, subsampling=0)),
    (1, 37, dict(quality=90, subsampling=2)), (37, 1, dict(quality=90, subsampling=1)),
    (2, 2, dict(quality=100, subsampling=2)), (5, 3, dict(quality=95, subsampling=2)),
    (9, 4, dict(quality=95, subsampling=1)), (6, 5, dict(quality=60, subsampling=2)),
    (17, 33, dict(quality=1, subsampling=2)), (31, 47, dict(quality=10, subsampling=1)),
    (64, 48, dict(quality=50, subsampling=0)), (23, 71, dict(quality=100, subsampling=0)),
    (57, 41, dict(quality=85, subsampling=2, optimize=True)), (40, 90, dict(quality=92, subsampling=1, optimize=True)),
    (45, 61, dict(quality=80, subsampling=2, restart_marker_blocks=1)),
    (33, 80, dict(quality=70, subsampling=0, restart_marker_blocks=5)),
    (70, 35, dict(quality=90, subsampling=1, restart_marker_rows=1)),
    (48, 48, dict(quality=99, subsampling=2, restart_marker_rows=2, optimize=True)),
    (29, 43, dict(quality=85, mode='L')), (1, 9, dict(quality=30, mode='L')),
    (40, 33, dict(quality=95, mode='L', restart_marker_blocks=3)),
    (300, 400, dict(quality=90, subsampling=2)), (401, 299, dict(quality=75, subsampling=1)),
]


def encode(h, w, seed=0, mode='RGB', **opts):
    img = PIL.fromarray(synth.photo_like_image(h, w, seed))
    if mode == 'L':
        img = img.convert('L')
    b = io.BytesIO()
    img.save(b, 'JPEG', **opts)
    return b.getvalue()


def pillow(data):
    return np.asarray(PIL.open(io.BytesIO(data)).convert('RGB'))


@pytest.mark.parametrize('i', range(len(CORPUS)))
def test_reference_equals_pillow(i):
    h, w, opts = CORPUS[i]
    data = encode(h, w, seed=i, **opts)
    route, hdr = jr.parse(data)
    assert route == 'gpu', hdr
    np.testing.assert_array_equal(jr.decode(data), pillow(data))


def test_reference_equals_pillow_over_every_quality():
    for q in range(1, 101, 3):
        data = encode(24, 40, seed=q, quality=q, subsampling=q % 3)
        np.testing.assert_array_equal(jr.decode(data), pillow(data), err_msg=f'quality {q}')


@pytest.mark.parametrize('opts', [dict(subsampling=2), dict(subsampling=0, restart_marker_blocks=3),
                                  dict(subsampling=1, optimize=True), dict(mode='L', restart_marker_rows=1)])
def test_self_synchronising_decode_equals_serial(opts):
    data = encode(40, 56, seed=3, quality=90, **opts)
    _, hdr = jr.parse(data)
    buf, starts = jr.unstuff(data, hdr['seg'])
    want = jr.coefficients_serial(hdr, buf, starts)
    for S in (16, 64, 256, 1024):
        n_subs = len(jr.subsequences(hdr, buf, starts, S))
        for cap in (0, 1, 2, 64):
            got, rounds, fallbacks = jr.self_sync(hdr, buf, starts, S, cap)
            np.testing.assert_array_equal(got, want, err_msg=f'S {S} cap {cap}')
            assert rounds <= cap
            if cap == 0:
                assert fallbacks == n_subs
    np.testing.assert_array_equal(jr.decode(data, S=64, max_rounds=3), pillow(data))


def test_streams_the_gpu_does_not_decode_go_to_pillow():
    img = PIL.fromarray(synth.photo_like_image(24, 32, 1))
    b = io.BytesIO()
    img.save(b, 'JPEG', progressive=True)
    assert jr.parse(b.getvalue()) == ('pillow', 'SOF2')
    b = io.BytesIO()
    img.convert('CMYK').save(b, 'JPEG')
    assert jr.parse(b.getvalue())[0] == 'pillow'
    # Adobe RGB: an APP14 segment with transform 0 in front of a YCbCr-sampled frame
    data = encode(24, 32, quality=90, subsampling=0)
    adobe = b'\xff\xee\x00\x0eAdobe\x00\x64\x00\x00\x00\x00\x00'
    assert jr.parse(data[:2] + adobe + data[2:]) == ('pillow', 'Adobe transform 0')
    assert jr.parse(data[:2] + adobe[:-1] + b'\x01' + data[2:])[0] == 'gpu'
    # 4:4:0 (luma 1x2): the SOF's sampling bytes edited; parsed only
    data = bytearray(encode(24, 32, quality=90, subsampling=0))
    sof = data.index(b'\xff\xc0')
    assert data[sof + 11] == 0x11
    data[sof + 11] = 0x12
    route, why = jr.parse(bytes(data))
    assert route == 'pillow' and why.startswith('sampling')


def without(data, marker):
    """data with every segment of the given marker removed"""
    while marker in data:
        i = data.index(marker)
        data = data[:i] + data[i + 2 + ((data[i + 2] << 8) | data[i + 3]):]
    return data


def all_ones_huffman(data):
    """data with codes added to its first Huffman table until one code is all ones (libjpeg refuses that table)"""
    i = data.index(b'\xff\xc4')
    ln = (data[i + 2] << 8) | data[i + 3]
    seg = data[i + 4:i + 2 + ln]
    bits = list(seg[1:17])
    cnt = sum(bits)
    longest = max(k + 1 for k, b in enumerate(bits) if b)
    add = (1 << longest) - sum(b << (longest - k - 1) for k, b in enumerate(bits[:longest]))
    bits[longest - 1] += add
    new = seg[:1] + bytes(bits) + seg[17:17 + cnt] + bytes(add) + seg[17 + cnt:]
    return data[:i] + b'\xff\xc4' + (len(new) + 2).to_bytes(2, 'big') + new + data[i + 2 + ln:]


def swapped_scan_order(data):
    """the SOS of a three-component stream listing Cr before Cb: legal for libjpeg (blocks in scan order, colour in
    frame order)"""
    data = bytearray(data)
    s = data.index(b'\xff\xda') + 5
    data[s + 2:s + 4], data[s + 4:s + 6] = data[s + 4:s + 6], data[s + 2:s + 4]
    return bytes(data)


def test_streams_pillow_decodes_differently_go_to_pillow():
    """no DHT (libjpeg-turbo loads its standard tables, as for Motion-JPEG frames: Pillow decodes it) and a scan order
    other than the frame order (libjpeg's business, whatever it makes of it) take Pillow's route"""
    data = encode(40, 48, quality=90, subsampling=2)
    no_dht = without(data, b'\xff\xc4')
    assert jr.parse(no_dht) == ('pillow', 'Huffman table not defined')
    np.testing.assert_array_equal(pillow(no_dht), pillow(data))
    swapped = swapped_scan_order(encode(24, 32, quality=90, subsampling=0))
    assert jr.parse(swapped) == ('pillow', 'scan order differs from frame order')


def test_malformed_streams_are_refused():
    data = encode(40, 48, quality=90, subsampling=2)
    with pytest.raises(jr.JpegError, match='truncated'):
        jr.parse(data[:len(data) // 2])
    with pytest.raises(jr.JpegError, match='quantisation table missing'):
        jr.parse(without(data, b'\xff\xdb'))
    with pytest.raises(jr.JpegError, match='bad Huffman table'):
        jr.parse(all_ones_huffman(data))
    for bad in (data[:len(data) // 2], without(data, b'\xff\xdb'), all_ones_huffman(data)):
        with pytest.raises(OSError):                 # Pillow refuses them too
            PIL.open(io.BytesIO(bad)).convert('RGB')
    with pytest.raises(jr.JpegError, match='capacity'):
        jr.parse(data, max_pixels=40 * 48 - 1)
    jr.parse(data, max_pixels=40 * 48)
    with pytest.raises(jr.JpegError, match='SOI'):
        jr.parse(b'\x89PNG' + data[4:])
