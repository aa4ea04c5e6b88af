"""CPU: the restatement of the GPU JPEG decoder (tests/jpeg_ref.py) on streams Pillow's encoder does not write
(tests/jpeg_streams.py): damaged scans with the EOI kept, restart markers missing, repeated or renumbered, trailers,
table placement, colour-space signalling and re-encoded scans.  A stream Pillow decodes and the restatement routes to
the GPU decodes bit for bit like Pillow; a stream Pillow refuses is refused or routed to Pillow, which raises as the
reference's loader does; the self-synchronising decode equals libjpeg's serial loop on every damaged stream."""
import io

import numpy as np
import pytest

import jpeg_ref as jr
import jpeg_streams as js

PIL = pytest.importorskip('PIL.Image')
STREAMS = js.corpus()


def pillow(data):
    return np.asarray(PIL.open(io.BytesIO(data)).convert('RGB'))


@pytest.mark.parametrize('name', sorted(STREAMS))
def test_stream_equals_pillow_or_takes_the_pillow_route(name):
    data = STREAMS[name]
    try:
        want = pillow(data)
    except OSError:
        want = None
    try:
        route, hdr = jr.parse(data)
    except jr.JpegError:
        assert want is None, 'the GPU route refuses a stream Pillow decodes'
        return
    if want is None:
        assert route == 'pillow', 'the GPU route decodes a stream Pillow refuses'
        with pytest.raises(OSError):
            pillow(data)
        return
    if route == 'gpu':
        np.testing.assert_array_equal(jr.decode(data), want)


def expected_route(name):
    """the route each corpus stream takes: 'refused' by Pillow (a JFIF APP0 of 5 or 6 bytes), 'pillow' for the colour
    signals the GPU does not decode (Adobe transform 0; R, G, B component ids with neither a JFIF APP0 of 14 bytes nor
    an Adobe segment), 'gpu' for every other stream"""
    if not name.startswith('colour_'):
        return 'gpu'
    app0 = int(name.split('_')[2])
    if app0 in (5, 6):
        return 'refused'
    if name.endswith('_adobe_0') or ('_ids_82_71_66_' in name and name.endswith('_adobe_None') and app0 < 14):
        return 'pillow'
    return 'gpu'


def test_routes_of_the_corpus():
    """a routing change cannot shrink the comparison unnoticed: every stream takes the route listed for it"""
    got = {}
    for name, data in STREAMS.items():
        try:
            pillow(data)
            got[name] = jr.parse(data)[0]
        except OSError:
            got[name] = 'refused'
    assert got == {name: expected_route(name) for name in STREAMS}
    assert sum(r == 'gpu' for r in got.values()) == 125


@pytest.mark.parametrize('name', js.DAMAGED)
def test_self_synchronising_decode_equals_serial_on_damaged_streams(name):
    data = STREAMS[name]
    route, hdr = jr.parse(data)
    assert route == 'gpu'
    buf, starts = jr.unstuff(data, hdr['seg'])
    want = jr.coefficients_serial(hdr, buf, starts)
    for S in (16, 64, 1024):
        for cap in (0, 1, 64):
            got, rounds, _ = jr.self_sync(hdr, buf, starts, S, cap)
            np.testing.assert_array_equal(got, want, err_msg=f'S {S} cap {cap}')
            assert rounds <= cap


def test_interval_segments_follow_libjpeg_resync():
    """interval i > 0 expects RST((i - 1) mod 8): the segment after each marker it takes, -1 for an empty one"""
    rst = [0xD0 + (k & 7) for k in range(10)]
    assert jr.interval_segments(11, rst) == list(range(11))
    # RST1 missing: RST2 is one ahead of RST1, left unread (empty interval 2), then taken for interval 3
    assert jr.interval_segments(6, [0xD0, 0xD2, 0xD3, 0xD4]) == [0, 1, -1, 2, 3, 4]
    # RST1 -> RST3 (two ahead): left unread twice, taken by interval 4; interval 5 then skips the prior RST2 and RST3
    assert jr.interval_segments(6, [0xD0, 0xD3, 0xD2, 0xD3, 0xD4]) == [0, 1, -1, -1, 2, 5]
    # a prior marker (RST1 where RST3 is due) is skipped with its data; a far one (RST7 for RST3) is taken
    assert jr.interval_segments(5, [0xD0, 0xD1, 0xD2, 0xD1, 0xD3]) == [0, 1, 2, 3, 5]
    assert jr.interval_segments(5, [0xD0, 0xD1, 0xD2, 0xD7]) == [0, 1, 2, 3, 4]
    # the numbers wrap: RST1 is two ahead of RST7
    assert jr.interval_segments(10, rst[:7] + [0xD1]) == [0, 1, 2, 3, 4, 5, 6, 7, -1, -1]
    # a code below SOF0 is skipped; the scan's end leaves every later interval empty
    assert jr.interval_segments(4, [0xD0, 0x05, 0xD1]) == [0, 1, 3, -1]
    assert jr.interval_segments(3, []) == [0, -1, -1]


def test_scan_ends_at_the_first_marker_that_is_not_a_restart():
    """trailers after EOI, garbage before it and a whole second image are not part of the scan"""
    clean = js.b420()
    for name in ('trailer_with_markers', 'second_jpeg_after_eoi'):
        _, hdr = jr.parse(STREAMS[name])
        assert hdr['seg'] == jr.parse(clean)[1]['seg']
    _, hdr = jr.parse(STREAMS['fill_before_eoi'])
    assert STREAMS['fill_before_eoi'][hdr['seg'][1]:] == b'\xff\xff\xff\xd9'
    _, hdr = jr.parse(STREAMS['resync_non_rst_marker'])
    assert hdr['n_segments'] == 7 and hdr['int_seg'][7:] == [-1] * (hdr['n_intervals'] - 7)
    with pytest.raises(jr.JpegError, match='no EOI'):
        jr.parse(clean[:-2])
    with pytest.raises(jr.JpegError, match='no EOI'):
        jr.parse(STREAMS['cut_half_scan'][:-2] + b'\xff\xc4\x00\x02')


def test_corpus_reaches_the_shapes_it_names():
    def hdr_of(name):
        return jr.parse(STREAMS[name])[1]

    def coefs(name):
        hdr = hdr_of(name)
        buf, starts = jr.unstuff(STREAMS[name], hdr['seg'])
        return hdr, jr.coefficients_serial(hdr, buf, starts)
    # 16-bit codes; every AC symbol in one table; one table pair per component
    assert any(int(t['maxcode'][16]) >= 0 for c in hdr_of('enc_skewed_16bit')['comps'] for t in (c['dc'], c['ac']))
    assert hdr_of('enc_skewed_16bit')['ri'] == 5
    assert all(int(c['ac']['maxcode'][16]) >= 0 for c in hdr_of('enc_all_162_symbols')['comps'])
    assert len({id(c['dc']) for c in hdr_of('enc_separate_tables')['comps']}) == 3
    # DC differences of category 11 and AC values of category 10
    hdr, c = coefs('enc_impulses_q100')
    nb = len(hdr['blocks'])
    y = c.reshape(-1, nb, 64)[:, 0, 0]
    assert np.abs(np.diff(y)).max() >= 1024 and np.abs(c[:, 1:]).max() >= 512
    # blocks over the IDCT's 16-bit lanes: a DC-only block with a dequantised DC of 8192 or more (pass 1's shortcut
    # wraps), and in0 + in4 over 16 bits in a block with more than row 0
    hdr, c = coefs('enc_idct_lanes')
    q = hdr['comps'][0]['q']
    luma = np.concatenate([np.arange(m * len(hdr['blocks']), m * len(hdr['blocks']) + 4)
                           for m in range(hdr['mx'] * hdr['my'])])
    x = c[luma] * q
    dc_only = ~(c[luma][:, 8:] != 0).any(1)
    assert (dc_only & (np.abs(x[:, 0]) >= 8192)).any()
    assert (~dc_only & (np.abs(x[:, 0] + x[:, 32]) > 32767)).any()
    # runs that end at k = 63
    hdr, c = coefs('enc_run_to_63_zrl_eob')
    assert (c[:, 63] != 0).sum() > 10
    # restarts every 1, 7 and 8 MCUs at every sampling, sizes off the MCU grid
    for ri in (1, 7, 8):
        for sub in (0, 1, 2, 'L'):
            hdr = hdr_of(f'enc_restart_{ri}_{sub}')
            assert hdr['ri'] == ri and hdr['n_intervals'] > 1 and (hdr['w'] % 8 or hdr['h'] % 8)
    # damaged scans starve: some blocks of the serial decode are left uniform grey
    for name in ('cut_half_scan', 'cut_inside_interval', 'cut_after_rst', 'missing_middle_rst', 'resync_next_plus_2'):
        hdr, c = coefs(name)
        assert (np.abs(c).sum(1) == 0).any(), name


def test_pillow_refused_streams_stay_refused():
    """JFIF / Adobe segments too short for Pillow's parser: the restatement routes them to Pillow, which raises"""
    refused = [n for n in STREAMS if n.startswith(('colour_app0_5_', 'colour_app0_6_'))]
    assert len(refused) == 18
    for n in refused:
        assert jr.parse(STREAMS[n]) == ('pillow', 'JFIF segment Pillow cannot parse')
        with pytest.raises(OSError):
            pillow(STREAMS[n])
    d = js.b420()
    short_adobe = d[:2] + b'\xff\xee\x00\x07Adobe' + d[2:]
    assert jr.parse(short_adobe)[0] == 'pillow'
    with pytest.raises(OSError):
        pillow(short_adobe)
