"""A seeded corpus of JPEG streams beyond Pillow's encoder, for tests/test_jpeg_streams*.py.

Each generator is a small named function returning bytes, built from Pillow-encoded streams by byte edits or by a
small Huffman re-encoder (`reencode`: coefficients from the restatement's serial decode, written again with chosen
tables and restart interval).  Families: damaged entropy data with the EOI kept, restart markers missing, repeated or
renumbered (one case per decision of libjpeg's jpeg_resync_to_restart), containers (trailers, Exif thumbnails, marker
bytes in segments, table placement, 16-bit DQT, colour-space signalling) and encoder shapes Pillow never writes."""
import heapq
import io

import numpy as np

import jpeg_ref as jr
from openpifpaf_b200 import synth

EOI = b'\xff\xd9'


def encode(h, w, seed=0, mode='RGB', image=None, **opts):
    from PIL import Image
    img = Image.fromarray(synth.photo_like_image(h, w, seed) if image is None else image)
    if mode == 'L':
        img = img.convert('L')
    b = io.BytesIO()
    img.save(b, 'JPEG', **opts)
    return b.getvalue()


def scan_start(data):
    i = data.index(b'\xff\xda')
    return i + 2 + ((data[i + 2] << 8) | data[i + 3])


def rst_positions(data):
    """offsets of the FF of every RSTn in the scan of a clean stream"""
    s, e = scan_start(data), len(data) - 2
    return [i for i in range(s, e - 1) if data[i] == 0xFF and 0xD0 <= data[i + 1] <= 0xD7]


def segments(data):
    """[(marker, whole segment bytes)] from SOI up to (not including) the SOS, and the rest from the SOS on"""
    out, pos = [], 2
    while data[pos + 1] != 0xDA:
        ln = (data[pos + 2] << 8) | data[pos + 3]
        out.append((data[pos + 1], data[pos:pos + 2 + ln]))
        pos += 2 + ln
    return out, data[pos:]


def assemble(segs, rest):
    return b'\xff\xd8' + b''.join(s for _, s in segs) + rest


def segment(marker, payload):
    return bytes([0xFF, marker]) + (len(payload) + 2).to_bytes(2, 'big') + payload


def rng(seed):
    return np.random.default_rng(seed)


def random_bytes(seed, n, allow_ff=True):
    b = rng(seed).integers(0, 256 if allow_ff else 255, n, dtype=np.uint8)
    return bytes(b)


# ------------------------------------------------------------------------------------------------------ re-encoder
def huffman_bits(freq, symbols):
    """JPEG Annex K.2 / K.3: code lengths from frequencies, limited to 16 bits, the all-ones code reserved.
    -> (bits[16], symbols ordered by code length)"""
    heap = [(f, i, [s]) for i, (s, f) in enumerate(zip(symbols, freq))] + [(0, -1, [None])]
    heapq.heapify(heap)
    length = {s: 0 for s in symbols}
    length[None] = 0
    tie = len(symbols)
    while len(heap) > 1:
        fa, _, a = heapq.heappop(heap)
        fb, _, b = heapq.heappop(heap)
        for s in a + b:
            length[s] += 1
        tie += 1
        heapq.heappush(heap, (fa + fb, tie, a + b))
    bits = [0] * 40
    for s, ln in length.items():
        bits[ln] += 1
    for i in range(39, 16, -1):
        while bits[i] > 0:
            j = i - 2
            while bits[j] == 0:
                j -= 1
            bits[i] -= 2
            bits[i - 1] += 1
            bits[j + 1] += 2
            bits[j] -= 1
    i = 16
    while bits[i] == 0:
        i -= 1
    bits[i] -= 1                                   # the reserved code point
    order = sorted(symbols, key=lambda s: (-freq[symbols.index(s)], s))
    return bits[1:17], order


def skewed_bits(symbols):
    """one code of each length 1.. (2.. for more than 16 symbols) up to 15, the rest 16 bits long"""
    n = len(symbols)
    if n <= 16:
        bits = [1] * (n - 1) + [0] * (16 - n) + [1]
    else:
        bits = [0] + [1] * 14 + [n - 14]
    return bits, list(symbols)


AC_SYMBOLS = [0x00, 0xF0] + [(r << 4) | s for r in range(16) for s in range(1, 11)]


def codes(bits, vals):
    out, code, p = {}, 0, 0
    for ln in range(1, 17):
        for _ in range(bits[ln - 1]):
            out[vals[p]] = (code, ln)
            code += 1
            p += 1
        code <<= 1
    return out


def nbits(v):
    return int(abs(v)).bit_length()


def block_symbols(row, zrl_eob):
    """AC (symbol, value, size) list of one block (natural order row)"""
    zz = [int(row[jr.ZIGZAG[k]]) for k in range(64)]
    out, run = [], 0
    for k in range(1, 64):
        v = zz[k]
        if v == 0:
            run += 1
            continue
        while run > 15:
            out.append((0xF0, 0, 0))
            run -= 16
        s = nbits(v)
        out.append(((run << 4) | s, v, s))
        run = 0
    if run:
        if zrl_eob and run >= 16:
            out.append((0xF0, 0, 0))
        out.append((0x00, 0, 0))
    return out


def reencode(data, ri=0, tables='optimal', separate=False, zrl_eob=False, edit=None):
    """data (a clean Pillow stream) written again: its coefficients (edited by edit(coef, hdr) if given), restart
    interval ri, Huffman tables 'optimal' (Annex K), 'skewed' (16-bit codes) or 'all162' (every AC symbol present,
    skewed), one DC / AC table pair per component (separate) or luma / chroma; zrl_eob: a ZRL before the EOB of
    blocks ending in 16 or more zeros"""
    route, hdr = jr.parse(data)
    assert route == 'gpu'
    buf, starts = jr.unstuff(data, hdr['seg'])
    coef = jr.coefficients_serial(hdr, buf, starts)
    if edit:
        edit(coef, hdr)
    nb, ncomp = len(hdr['blocks']), len(hdr['comps'])
    tab = [c if separate else min(c, 1) for c in range(ncomp)]
    n_mcu = hdr['mx'] * hdr['my']
    ri_eff = ri or n_mcu
    # symbols per block, DC predictors reset at every interval
    stream = []
    for m in range(n_mcu):
        if m % ri_eff == 0:
            pred = [0] * ncomp
            stream.append(None)
        for t, (ci, _, _) in enumerate(hdr['blocks']):
            row = coef[m * nb + t]
            d = int(row[0]) - pred[ci]
            pred[ci] = int(row[0])
            stream.append((tab[ci], nbits(d), d, block_symbols(row, zrl_eob)))
    freq = {}
    for e in stream:
        if e is None:
            continue
        freq.setdefault((0, e[0]), {}).setdefault(e[1], 0)
        freq[(0, e[0])][e[1]] += 1
        for sym, _, _ in e[3]:
            freq.setdefault((1, e[0]), {}).setdefault(sym, 0)
            freq[(1, e[0])][sym] += 1
    dht, book = b'', {}
    for (kind, th) in sorted(freq):
        f = freq[(kind, th)]
        syms = sorted(f) if not (kind and tables == 'all162') else AC_SYMBOLS
        fr = [f.get(s, 0) for s in syms]
        if tables == 'optimal':
            bits, vals = huffman_bits(fr, syms)
        else:
            bits, vals = skewed_bits(sorted(syms, key=lambda s: (-f.get(s, 0), s)))
        book[(kind, th)] = codes(bits, vals)
        dht += bytes([(kind << 4) | th]) + bytes(bits) + bytes(vals)
    # entropy-coded data
    out, acc, nacc, rst = bytearray(), 0, 0, 0

    def put(code, ln):
        nonlocal acc, nacc
        acc = (acc << ln) | code
        nacc += ln
        while nacc >= 8:
            b = (acc >> (nacc - 8)) & 255
            out.append(b)
            if b == 0xFF:
                out.append(0)
            nacc -= 8
        acc &= (1 << nacc) - 1

    for i, e in enumerate(stream):
        if e is None:
            if i:
                if nacc:
                    put((1 << (8 - nacc)) - 1, 8 - nacc)
                out += bytes([0xFF, 0xD0 + rst])
                rst = (rst + 1) & 7
            continue
        th, s, d, acs = e
        put(*book[(0, th)][s])
        if s:
            put(d if d > 0 else d + (1 << s) - 1, s)
        for sym, v, sz in acs:
            put(*book[(1, th)][sym])
            if sz:
                put(v if v > 0 else v + (1 << sz) - 1, sz)
    if nacc:
        put((1 << (8 - nacc)) - 1, 8 - nacc)
    segs, rest = segments(data)
    segs = [(m, s) for m, s in segs if m not in (0xC4, 0xDD)]
    segs.append((0xC4, segment(0xC4, dht)))
    if ri:
        segs.append((0xDD, segment(0xDD, ri.to_bytes(2, 'big'))))
    sos = bytes([ncomp]) + b''.join(bytes([c['id'], (tab[k] << 4) | tab[k]]) for k, c in enumerate(hdr['comps']))
    return assemble(segs, segment(0xDA, sos + b'\x00\x3f\x00') + bytes(out) + EOI)


# ---------------------------------------------------------------------------------------------------- base streams
def b420():
    return encode(40, 56, seed=3, quality=90, subsampling=2)


def r1():
    """45 x 61 4:2:0, a restart every MCU (24 intervals: the RST numbers wrap three times)"""
    return encode(45, 61, seed=2, quality=80, subsampling=2, restart_marker_blocks=1)


def r3():
    return encode(48, 72, seed=5, quality=85, subsampling=0, restart_marker_blocks=3)


def cut_scan(data, at):
    """the scan cut `at` bytes after its start, EOI kept"""
    return data[:scan_start(data) + at] + EOI


# ------------------------------------------------------------------------------------------------- damaged scans
def cut_half_scan():
    d = b420()
    return cut_scan(d, (len(d) - 2 - scan_start(d)) // 2)


def cut_half_scan_trailer():
    return cut_half_scan() + random_bytes(11, 300) + EOI


def cut_inside_interval():
    d = r3()
    p = rst_positions(d)
    return d[:(p[3] + p[4]) // 2] + EOI


def cut_after_rst():
    d = r3()
    return d[:rst_positions(d)[4] + 2] + EOI


def cut_between_ff_00():
    d = b420()
    s = scan_start(d)
    i = d.index(b'\xff\x00', s + (len(d) - s) // 3)
    return d[:i + 1] + EOI


def cut_in_last_mcu():
    d = b420()
    return d[:-2 - 3] + EOI


def cut_at_scan_start():
    return cut_scan(b420(), 0)


def cut_at_scan_start_restarts():
    return cut_scan(r3(), 0)


def flip(data, n, seed):
    """n seeded bytes of the scan changed, no marker made or broken"""
    d = bytearray(data)
    s, r = scan_start(d), rng(seed)
    for i in r.choice(np.arange(s, len(d) - 2), n, replace=False):
        if d[i] != 0xFF and d[i - 1] != 0xFF:
            d[i] ^= int(r.integers(1, 256))
            d[i] = 0xFE if d[i] == 0xFF else d[i]
    return bytes(d)


def flipped_bytes():
    return flip(r3(), 6, 21)


def flipped_low_quality(q, seed):
    """12 flipped bytes in a 40 x 56 4:2:0 scan at quality q: coarse quantisation makes the damaged blocks overshoot
    the 16-bit lanes of the IDCT"""
    return flip(encode(40, 56, seed=seed, quality=q, subsampling=2), 12, 1000 + seed)


def flipped_bytes_no_restart():
    d = bytearray(b420())
    s = scan_start(d)
    for i in (s + 40, s + 41, s + 300):
        d[i] = 0x5A if d[i] != 0x5A else 0xA5
    return bytes(d)


def garbage_before_rst():
    d = r3()
    i = rst_positions(d)[2]
    return d[:i] + random_bytes(12, 40, allow_ff=False) + d[i:]


def garbage_before_eoi():
    d = b420()
    return d[:-2] + random_bytes(13, 25, allow_ff=False) + EOI


# ---------------------------------------------------------------------------------------------- restart markers
def drop_rst(k, data=None):
    d = data or r1()
    i = rst_positions(d)[k]
    return d[:i] + d[i + 2:]


def renumber_rst(k, delta, data=None):
    """RST number k (0-based) given the number of the marker expected there plus delta (mod 8)"""
    d = bytearray(data or r1())
    i = rst_positions(bytes(d))[k]
    d[i + 1] = 0xD0 + ((d[i + 1] - 0xD0 + delta) & 7)
    return bytes(d)


def missing_first_rst():
    return drop_rst(0)


def missing_middle_rst():
    return drop_rst(1)


def missing_last_rst():
    return drop_rst(len(rst_positions(r1())) - 1)


def duplicated_rst():
    d = r1()
    i = rst_positions(d)[5]
    return d[:i + 2] + d[i:i + 2] + d[i + 2:]


def resync_next_plus_1():
    return renumber_rst(1, 1)


def resync_next_plus_2():
    return renumber_rst(1, 2)


def resync_prior_minus_1():
    return renumber_rst(3, -1)


def resync_prior_minus_2():
    return renumber_rst(3, -2)


def resync_far():
    return renumber_rst(3, 4)


def resync_wraps():
    """RST7 renumbered RST1: two past the expected number, across the wrap"""
    return renumber_rst(7, 2)


def resync_non_rst_marker():
    d = bytearray(r1())
    i = rst_positions(bytes(d))[6]
    d[i + 1] = 0xD9
    return bytes(d)


def resync_invalid_marker():
    """FF 05 (below SOF0) in place of a restart marker: skipped with the data after it"""
    d = bytearray(r1())
    i = rst_positions(bytes(d))[6]
    d[i + 1] = 0x05
    return bytes(d)


def rst_without_dri():
    segs, rest = segments(r1())
    return assemble([(m, s) for m, s in segs if m != 0xDD], rest)


def set_dri(v):
    segs, rest = segments(r1())
    return assemble([(m, segment(0xDD, v.to_bytes(2, 'big')) if m == 0xDD else s) for m, s in segs], rest)


def dri_over_mcu_count():
    return set_dri(1000)


def dri_zero():
    return set_dri(0)


def fill_before_rst():
    d = r1()
    i = rst_positions(d)[3]
    return d[:i] + b'\xff\xff' + d[i:]


def fill_before_eoi():
    return r1()[:-2] + b'\xff\xff' + EOI


# ---------------------------------------------------------------------------------------------------- containers
def trailer_with_markers():
    t = bytearray(random_bytes(14, 500))
    for k, m in enumerate((0xD9, 0xD0, 0xD3, 0xD7, 0xD9)):
        t[60 * k + 7:60 * k + 9] = bytes([0xFF, m])
    return b420() + bytes(t)


def second_jpeg_after_eoi():
    return b420() + encode(24, 32, seed=9, quality=70, subsampling=1)


def exif_thumbnail():
    thumb = encode(16, 24, seed=4, quality=60, subsampling=2)
    ifd0 = (0).to_bytes(2, 'little') + (26).to_bytes(4, 'little')   # no entries, IFD1 at offset 26 (8 + 2 + 4 + 12)
    ifd1 = (2).to_bytes(2, 'little')
    ifd1 += (0x0201).to_bytes(2, 'little') + (4).to_bytes(2, 'little') + (1).to_bytes(4, 'little') + (56).to_bytes(4, 'little')
    ifd1 += (0x0202).to_bytes(2, 'little') + (4).to_bytes(2, 'little') + (1).to_bytes(4, 'little') + len(thumb).to_bytes(4, 'little')
    ifd1 += (0).to_bytes(4, 'little')
    tiff = b'II*\x00' + (8).to_bytes(4, 'little') + ifd0 + bytes(12) + ifd1
    tiff += bytes(56 - len(tiff)) + thumb
    d = b420()
    return d[:2] + segment(0xE1, b'Exif\x00\x00' + tiff) + d[2:]


def segments_holding_markers():
    d = r1()
    junk = b'\xff\xd9\xff\xd8\xff\xda\x00\x02\xff\xd0\xff\xc4'
    return d[:2] + segment(0xFE, junk) + segment(0xE5, junk + b'\xff') + d[2:]


def tables_after_frame():
    segs, rest = segments(b420())
    sof = [x for x in segs if x[0] == 0xC0]
    return assemble([x for x in segs if x[0] != 0xC0 and x[0] not in (0xDB, 0xC4)] + sof +
                    [x for x in segs if x[0] in (0xDB, 0xC4)], rest)


def tables_in_one_segment():
    segs, rest = segments(b420())
    dqt = b''.join(s[4:] for m, s in segs if m == 0xDB)
    dht = b''.join(s[4:] for m, s in segs if m == 0xC4)
    keep = [x for x in segs if x[0] not in (0xDB, 0xC4)]
    return assemble(keep[:1] + [(0xDB, segment(0xDB, dqt)), (0xC4, segment(0xC4, dht))] + keep[1:], rest)


def tables_redefined():
    """every DQT and DHT given first with other contents (the chroma tables in the luma slots and back), then again
    as written before the SOS"""
    segs, rest = segments(b420())
    dqt = [s for m, s in segs if m == 0xDB]
    dht = [s for m, s in segs if m == 0xC4]
    swap = bytearray(b''.join(s[4:] for s in dht))
    i = 0
    while i < len(swap):                              # table ids 0 <-> 1
        swap[i] ^= 1
        i += 17 + sum(swap[i + 1:i + 17])
    qs = bytearray(b''.join(s[4:] for s in dqt))
    for j in range(0, len(qs), 65):
        qs[j] ^= 1
    early = [(0xDB, segment(0xDB, bytes(qs))), (0xC4, segment(0xC4, bytes(swap)))]
    return assemble(segs[:1] + early + segs[1:], rest)


def sof1_16bit_dqt():
    q = [[40000] * 64, [3 * v for v in range(1, 65)]]
    return encode(40, 56, seed=5, qtables=q, subsampling=2)


def colour_signal(app0_len, ids, adobe):
    """24 x 32 4:4:4 with a JFIF APP0 of app0_len data bytes (0: none), component ids, Adobe transform (None: no
    APP14)"""
    segs, rest = segments(encode(24, 32, seed=1, quality=90, subsampling=0))
    segs = [x for x in segs if x[0] != 0xE0]
    out = []
    if app0_len:
        out.append((0xE0, segment(0xE0, (b'JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00\x00\x00')[:app0_len])))
    if adobe is not None:
        out.append((0xEE, segment(0xEE, b'Adobe\x00\x64\x00\x00\x00\x00' + bytes([adobe]))))
    for m, s in segs:
        if m == 0xC0:
            s = bytearray(s)
            for k, cid in enumerate(ids):
                s[10 + 3 * k] = cid
            s = bytes(s)
        out.append((m, s))
    rest = bytearray(rest)
    for k, cid in enumerate(ids):
        rest[5 + 2 * k] = cid
    return assemble(out, bytes(rest))


# ------------------------------------------------------------------------------------------------ encoder shapes
def impulses(h, w):
    """black and white 8 x 8 blocks (DC differences of category 11), shifted by half a block in the lower half (a
    step across every block: AC values of category 10), and single green pixels"""
    img = np.zeros((h, w, 3), dtype=np.uint8)
    yy, xx = np.mgrid[0:h, 0:w]
    shift = np.where(yy >= h // 2, 4, 0)
    img[((yy // 8 + (xx + shift) // 8) % 2 == 0)] = 255
    img[4::16, 4::16] = (0, 255, 0)
    return img


def run_to_63(coef, hdr):
    coef[::3, 63] = 1
    coef[1::5, 63] = -3


def idct_lanes(coef, hdr):
    """luma blocks that reach each 16-bit lane of libjpeg-turbo's SIMD islow IDCT (dequantised values in brackets):
    DC-only blocks [8193, -12000, 6000] whose pass-1 shortcut shifts in 16 bits; in0 + in4 [8193 + 26000],
    in5 + in1 and in7 + in3 [17000 each] over 16 bits in pass 1; row 0 only with (0, 3) and (0, 7) [6000 each]: a
    workspace whose in7 + in3 wraps in pass 2; (0, 0) and (0, 4) [6000 each] with a small (1, 1): the same for
    in0 + in4; a product (2, 2) [40000] over 16 bits"""
    q, nb = hdr['comps'][0]['q'], len(hdr['blocks'])
    luma = [m * nb + t for m in range(hdr['mx'] * hdr['my']) for t in range(4)]
    cases = [{0: 8193}, {0: -12000}, {0: 6000}, {0: 8193, 32: 26000}, {8: 17000, 40: 17000},
             {24: 17000, 56: 17000}, {3: 6000, 7: 6000}, {0: 6000, 4: 6000, 9: 40}, {18: 40000}]
    for b, case in zip(luma[1::2], cases):
        coef[b] = 0
        for idx, target in case.items():
            coef[b, idx] = int(np.sign(target)) * -(-abs(target) // int(q[idx]))


def enc_idct_lanes():
    return reencode(encode(32, 48, seed=10, quality=90, subsampling=2), edit=idct_lanes)


def enc_separate_tables():
    return reencode(encode(41, 59, seed=6, quality=85, subsampling=2), separate=True)


def enc_skewed_16bit():
    return reencode(encode(37, 45, seed=7, quality=75, subsampling=1), tables='skewed', ri=5)


def enc_all_162_symbols():
    return reencode(encode(33, 47, seed=8, quality=95, subsampling=0), tables='all162', separate=True)


def enc_run_to_63_zrl_eob():
    return reencode(encode(40, 40, seed=9, quality=60, subsampling=2), edit=run_to_63, zrl_eob=True)


def enc_impulses_q100():
    return reencode(encode(48, 64, image=impulses(48, 64), quality=100, subsampling=0), ri=7)


def enc_restarts(ri, sub):
    h, w = {0: (27, 35), 1: (29, 37), 2: (47, 61), 'L': (23, 41)}[sub]
    opts = dict(mode='L') if sub == 'L' else dict(subsampling=sub)
    return reencode(encode(h, w, seed=20 + ri, quality=88, **opts), ri=ri)


# -------------------------------------------------------------------------------------------------------- corpus
def corpus():
    """{name: bytes}"""
    out = {}
    for f in (cut_half_scan, cut_half_scan_trailer, cut_inside_interval, cut_after_rst, cut_between_ff_00,
              cut_in_last_mcu, cut_at_scan_start, cut_at_scan_start_restarts, flipped_bytes,
              flipped_bytes_no_restart, garbage_before_rst, garbage_before_eoi,
              missing_first_rst, missing_middle_rst, missing_last_rst, duplicated_rst, resync_next_plus_1,
              resync_next_plus_2, resync_prior_minus_1, resync_prior_minus_2, resync_far, resync_wraps,
              resync_non_rst_marker, resync_invalid_marker, rst_without_dri, dri_over_mcu_count, dri_zero,
              fill_before_rst, fill_before_eoi,
              trailer_with_markers, second_jpeg_after_eoi, exif_thumbnail, segments_holding_markers,
              tables_after_frame, tables_in_one_segment, tables_redefined, sof1_16bit_dqt,
              enc_separate_tables, enc_skewed_16bit, enc_all_162_symbols, enc_run_to_63_zrl_eob, enc_impulses_q100, enc_idct_lanes):
        out[f.__name__] = f()
    for q in (5, 15, 30):
        for seed in range(4):
            out[f'flipped_low_quality_{q}_{seed}'] = flipped_low_quality(q, seed)
    for ri in (1, 7, 8):
        for sub in (0, 1, 2, 'L'):
            out[f'enc_restart_{ri}_{sub}'] = enc_restarts(ri, sub)
    for ln in range(0, 17):
        if 0 < ln < 5:
            continue
        for ids in ((1, 2, 3), (0, 1, 2), (82, 71, 66)):
            for adobe in (None, 0, 1):
                out[f'colour_app0_{ln}_ids_{"_".join(map(str, ids))}_adobe_{adobe}'] = colour_signal(ln, ids, adobe)
    return out


DAMAGED = [n for n in ('cut_half_scan', 'cut_half_scan_trailer', 'cut_inside_interval', 'cut_after_rst',
                       'cut_between_ff_00', 'cut_in_last_mcu', 'cut_at_scan_start', 'cut_at_scan_start_restarts',
                       'flipped_bytes', 'flipped_bytes_no_restart', 'garbage_before_rst', 'garbage_before_eoi',
                       'missing_first_rst', 'missing_middle_rst', 'missing_last_rst', 'duplicated_rst',
                       'resync_next_plus_1', 'resync_next_plus_2', 'resync_prior_minus_1', 'resync_prior_minus_2',
                       'resync_far', 'resync_wraps', 'resync_non_rst_marker', 'resync_invalid_marker',
                       'rst_without_dri', 'dri_over_mcu_count', 'dri_zero', 'fill_before_rst')] + \
    [f'flipped_low_quality_{q}_{seed}' for q in (5, 15, 30) for seed in range(4)]
