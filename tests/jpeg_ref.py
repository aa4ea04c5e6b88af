"""Python restatement of the GPU JPEG decoder (openpifpaf_b200/csrc/jpeg.cu) for the CPU tests.

Each step is the same integer arithmetic the kernels do, written for clarity rather than speed:
  parse              marker walk, routing ('gpu' / 'pillow') and validation, as pifpaf_jpeg_decode's host code
  huff_table         9-bit lookup + canonical maxcode / valoffset per DHT table
  unstuff            FF00 removal and restart-interval starts (k_jpeg_unstuff)
  decode_run         the Huffman decoder state machine over one interval (k_jpeg_sync / k_jpeg_write)
  self_sync          Weissenberger & Schmidt's self-synchronising decode, rounds capped, serial fallback
  idct_islow         libjpeg's jidctint (CONST_BITS 13, PASS1_BITS 2) with the post-IDCT range limit
  upsample_h2v1/h2v2 libjpeg-turbo's fancy upsamplers (jdsample.c)
  ycc_to_rgb         jdcolor.c's fixed-point tables (SCALEBITS 16)
`decode(data)` chains them into what `np.asarray(PIL.Image.open(data).convert('RGB'))` returns for 'gpu' streams.
"""
import numpy as np

ZIGZAG = np.array([
    0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21,
    28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61,
    54, 47, 55, 62, 63], dtype=np.int64)
LOOKUP_BITS = 9


class JpegError(ValueError):
    """A malformed or truncated stream, or one over the decoder's capacities."""


# ------------------------------------------------------------------------------------------------------------ parser
def huff_table(bits, vals, is_dc):
    """bits: counts of codes of length 1..16, vals: symbols -> dict(lookup [512] (len << 8 | sym, 0 = longer code),
    maxcode [18] (-1: no code of that length; [17] sentinel), valoffset [17], vals [256])"""
    if sum(bits) > 256 or len(vals) != sum(bits):
        raise JpegError('bad Huffman table')
    if is_dc and any(v > 15 for v in vals):
        raise JpegError('bad DC Huffman symbol')
    lookup = np.zeros(1 << LOOKUP_BITS, dtype=np.int32)
    maxcode = np.full(18, -1, dtype=np.int64)
    valoffset = np.zeros(17, dtype=np.int64)
    code, p = 0, 0
    for ln in range(1, 17):
        n = bits[ln - 1]
        if n:
            valoffset[ln] = p - code
            for i in range(n):
                if ln <= LOOKUP_BITS:
                    lo = code << (LOOKUP_BITS - ln)
                    lookup[lo:lo + (1 << (LOOKUP_BITS - ln))] = (ln << 8) | vals[p]
                code += 1
                p += 1
            maxcode[ln] = code - 1
        if code >= (1 << ln):                      # jpeg_make_d_derived_tbl: no code is all ones
            raise JpegError('bad Huffman table')
        code <<= 1
    maxcode[17] = 0xFFFFF
    v = np.zeros(256, dtype=np.int64)
    v[:len(vals)] = vals
    return dict(lookup=lookup, maxcode=maxcode, valoffset=valoffset, vals=v)


def parse(data, max_pixels=1 << 62):
    """-> ('pillow', reason) or ('gpu', header).  Raises JpegError on a malformed stream (the same checks as
    pifpaf_jpeg_decode, made before anything is launched)."""
    data = bytes(data)
    n = len(data)
    if n < 4 or data[0] != 0xFF or data[1] != 0xD8:
        raise JpegError('no SOI marker')
    pos = 2
    qt, dc, ac = {}, {}, {}
    frame, ri, jfif, adobe = None, 0, False, None
    while True:
        if pos >= n or data[pos] != 0xFF:
            raise JpegError('marker expected')
        while pos < n and data[pos] == 0xFF:
            pos += 1
        if pos >= n:
            raise JpegError('truncated marker')
        m = data[pos]
        pos += 1
        if m == 0xD9 or 0xD0 <= m <= 0xD7 or m == 0x01:
            if m == 0xD9:
                raise JpegError('EOI before the scan')
            continue
        if pos + 2 > n:
            raise JpegError('truncated segment length')
        ln = (data[pos] << 8) | data[pos + 1]
        if ln < 2 or pos + ln > n:
            raise JpegError('segment runs past the end of the stream')
        seg = data[pos + 2:pos + ln]
        pos += ln
        if m in (0xC0, 0xC1):
            if frame is not None:
                raise JpegError('second frame header')
            if len(seg) < 6:
                raise JpegError('short SOF')
            prec, h, w, nf = seg[0], (seg[1] << 8) | seg[2], (seg[3] << 8) | seg[4], seg[5]
            if len(seg) != 6 + 3 * nf:
                raise JpegError('bad SOF length')
            comps = [dict(id=seg[6 + 3 * i], h=seg[7 + 3 * i] >> 4, v=seg[7 + 3 * i] & 15, tq=seg[8 + 3 * i])
                     for i in range(nf)]
            frame = dict(prec=prec, h=h, w=w, comps=comps)
        elif 0xC2 <= m <= 0xCF and m not in (0xC4, 0xC8, 0xCC):
            return 'pillow', f'SOF{m - 0xC0}'
        elif m == 0xCC:
            return 'pillow', 'arithmetic coding'
        elif m == 0xC4:
            i = 0
            while i < len(seg):
                if i + 17 > len(seg):
                    raise JpegError('short DHT')
                tc, th = seg[i] >> 4, seg[i] & 15
                bits = list(seg[i + 1:i + 17])
                cnt = sum(bits)
                if tc > 1 or th > 3 or i + 17 + cnt > len(seg):
                    raise JpegError('bad DHT')
                (dc if tc == 0 else ac)[th] = huff_table(bits, list(seg[i + 17:i + 17 + cnt]), tc == 0)
                i += 17 + cnt
        elif m == 0xDB:
            i = 0
            while i < len(seg):
                pq, tq = seg[i] >> 4, seg[i] & 15
                sz = 128 if pq else 64
                if pq > 1 or tq > 3 or i + 1 + sz > len(seg):
                    raise JpegError('bad DQT')
                raw = np.frombuffer(seg[i + 1:i + 1 + sz], dtype='>u2' if pq else np.uint8).astype(np.int64)
                t = np.zeros(64, dtype=np.int64)
                t[ZIGZAG] = raw
                qt[tq] = t
                i += 1 + sz
        elif m == 0xDD:
            if len(seg) != 2:
                raise JpegError('bad DRI length')
            ri = (seg[0] << 8) | seg[1]
        elif m == 0xE0:
            jfif = jfif or seg[:5] == b'JFIF\x00'
        elif m == 0xEE:
            if seg[:5] == b'Adobe' and len(seg) >= 12:
                adobe = seg[11]
        elif m == 0xDA:
            return _scan(data, pos, seg, frame, qt, dc, ac, ri, jfif, adobe, max_pixels)
        # any other APPn / COM / DNL-free segment is skipped


def _scan(data, pos, seg, frame, qt, dc, ac, ri, jfif, adobe, max_pixels):
    if frame is None:
        raise JpegError('SOS before SOF')
    if len(seg) < 1 or len(seg) != 4 + 2 * seg[0]:
        raise JpegError('bad SOS length')
    comps, ns = frame['comps'], seg[0]
    h, w = frame['h'], frame['w']
    if frame['prec'] != 8:
        return 'pillow', f'{frame["prec"]}-bit samples'
    if len(comps) not in (1, 3):
        return 'pillow', f'{len(comps)} components'
    if len(comps) == 3:
        ids = tuple(c['id'] for c in comps)
        if adobe is not None and adobe != 1:
            return 'pillow', f'Adobe transform {adobe}'
        if not jfif and adobe is None and ids == (82, 71, 66):
            return 'pillow', 'RGB component ids'
        if (comps[1]['h'], comps[1]['v'], comps[2]['h'], comps[2]['v']) != (1, 1, 1, 1) or \
                (comps[0]['h'], comps[0]['v']) not in ((1, 1), (2, 1), (2, 2)):
            return 'pillow', 'sampling ' + ','.join(f'{c["h"]}x{c["v"]}' for c in comps)
    if ns != len(comps):
        return 'pillow', 'multi-scan'
    ss, se, ahal = seg[1 + 2 * ns], seg[2 + 2 * ns], seg[3 + 2 * ns]
    if (ss, se, ahal) != (0, 63, 0):
        raise JpegError('bad spectral selection for a sequential scan')
    if h == 0 or w == 0:
        raise JpegError('zero image size')
    if w * h > max_pixels:
        raise JpegError('image over capacity')
    order = []
    for i in range(ns):
        cid, tt = seg[1 + 2 * i], seg[2 + 2 * i]
        ci = [j for j, c in enumerate(comps) if c['id'] == cid]
        if len(ci) != 1 or ci[0] in order:
            raise JpegError('scan component not in the frame')
        order.append(ci[0])
        c = comps[ci[0]]
        if (tt >> 4) > 3 or (tt & 15) > 3:
            raise JpegError('bad Huffman table selector')
        if c['tq'] not in qt:
            raise JpegError('quantisation table missing')
        c['dc'], c['ac'] = dc.get(tt >> 4), ac.get(tt & 15)
        c['q'] = qt[c['tq']]
    # libjpeg-turbo fills an undefined Huffman slot with its standard tables (Motion-JPEG); libjpeg converts colour in
    # frame order and reads blocks in scan order: Pillow decodes both kinds of stream
    if any(c['dc'] is None or c['ac'] is None for c in comps):
        return 'pillow', 'Huffman table not defined'
    if order != list(range(ns)):
        return 'pillow', 'scan order differs from frame order'
    end = data.rfind(b'\xff\xd9')
    if end < pos:
        raise JpegError('no EOI after the scan (truncated stream)')
    comps = [comps[i] for i in order]
    if len(comps) == 1:
        comps[0]['h'] = comps[0]['v'] = 1          # a one-component scan is not interleaved: 1 block per MCU
    hmax, vmax = max(c['h'] for c in comps), max(c['v'] for c in comps)
    mx, my = -(-w // (8 * hmax)), -(-h // (8 * vmax))
    blocks = [(ci, bv, bh) for ci, c in enumerate(comps) for bv in range(c['v']) for bh in range(c['h'])]
    n_mcu = mx * my
    return 'gpu', dict(w=w, h=h, comps=comps, hmax=hmax, vmax=vmax, mx=mx, my=my, blocks=blocks, ri=ri or n_mcu,
                       n_intervals=-(-n_mcu // (ri or n_mcu)), seg=(pos, end))


# ------------------------------------------------------------------------------------------------------ entropy data
def unstuff(data, seg):
    """-> (compacted bytes, [start byte of each interval]).  FF00 -> FF; FF D0..D7 dropped and recorded."""
    s = data[seg[0]:seg[1]]
    out, starts = bytearray(), [0]
    i = 0
    while i < len(s):
        b = s[i]
        if b == 0xFF and i + 1 < len(s):
            nb = s[i + 1]
            if nb == 0x00:
                out.append(0xFF)
                i += 2
                continue
            if 0xD0 <= nb <= 0xD7:
                starts.append(len(out))
                i += 2
                continue
        out.append(b)
        i += 1
    return bytes(out), starts


class Bits:
    """bit reader over one interval: bits past its end read as zeros (libjpeg's behaviour at a marker)"""

    def __init__(self, buf, lo, hi):
        self.buf, self.lo, self.hi = buf, lo, hi

    def peek(self, pos, n):
        """n (<= 16) bits at bit offset pos of the interval"""
        i = self.lo + (pos >> 3)
        v = 0
        for k in range(3):
            v = (v << 8) | (self.buf[i + k] if i + k < self.hi else 0)
        return (v >> (24 - (pos & 7) - n)) & ((1 << n) - 1)


def huff_decode(tbl, bits, pos):
    """-> (symbol, code length)"""
    e = int(tbl['lookup'][bits.peek(pos, LOOKUP_BITS)])
    if e:
        return e & 255, e >> 8
    ln = LOOKUP_BITS + 1
    code = bits.peek(pos, ln)
    while ln <= 16 and code > tbl['maxcode'][ln]:
        ln += 1
        code = bits.peek(pos, ln) if ln <= 16 else code
    if ln > 16:
        return 0, 16                               # corrupt code: a zero symbol, like libjpeg
    return int(tbl['vals'][int(tbl['valoffset'][ln]) + code]), ln


def extend(v, s):
    return v - (1 << s) + 1 if s and v < (1 << (s - 1)) else v


def decode_run(hdr, bits, state, end_bit, emit=None, max_blocks=None):
    """Decode from state (bit, block in MCU, k) until the first codeword boundary at or after end_bit (or after
    max_blocks block starts).  emit(block_starts_so_far_minus_one, natural index, value) receives every coefficient
    (DC: the difference).  -> (exit state, number of block starts)"""
    pos, blk, k = state
    comps, blocks = hdr['comps'], hdr['blocks']
    bpm = len(blocks)
    nstart = 0
    while pos < end_bit:
        c = comps[blocks[blk][0]]
        if k == 0:
            if max_blocks is not None and nstart >= max_blocks:
                break
            s, ln = huff_decode(c['dc'], bits, pos)
            pos += ln
            v = extend(bits.peek(pos, s), s) if s else 0
            pos += s
            nstart += 1
            if emit:
                emit(nstart - 1, 0, v)
            k = 1
        else:
            rs, ln = huff_decode(c['ac'], bits, pos)
            pos += ln
            r, s = rs >> 4, rs & 15
            if s:
                k += r
                v = extend(bits.peek(pos, s), s)
                pos += s
                if emit:
                    emit(nstart - 1, int(ZIGZAG[min(k, 63)]), v)
                k += 1
            elif r == 15:
                k += 16
            else:
                k = 64
        if k >= 64:
            k = 0
            blk = (blk + 1) % bpm
    return (pos, blk, k), nstart


def interval_blocks(hdr, i):
    n_mcu = hdr['mx'] * hdr['my']
    lo = i * hdr['ri']
    return (min(lo + hdr['ri'], n_mcu) - lo) * len(hdr['blocks'])


def coefficients_serial(hdr, buf, starts):
    """int64 [n_blocks, 64] in scan order, DC resolved (the serial decode, libjpeg's order)"""
    nb = len(hdr['blocks'])
    coef = np.zeros((hdr['mx'] * hdr['my'] * nb, 64), dtype=np.int64)
    ends = list(starts[1:hdr['n_intervals']]) + [len(buf)]
    for i in range(hdr['n_intervals']):
        lo = starts[i] if i < len(starts) else len(buf)
        hi = ends[i] if i < len(ends) else len(buf)
        base, cnt = i * hdr['ri'] * nb, interval_blocks(hdr, i)

        def emit(b, z, v):
            coef[base + b, z] = v
        decode_run(hdr, Bits(buf, lo, hi), (0, 0, 0), 1 << 62, emit, max_blocks=cnt)
    resolve_dc(hdr, coef)
    return coef


def resolve_dc(hdr, coef):
    """DC differences -> DC values: a prefix sum per component, reset at every interval start"""
    nb = len(hdr['blocks'])
    comp_of = np.array([b[0] for b in hdr['blocks']])
    blk_comp = np.tile(comp_of, coef.shape[0] // nb)
    interval = np.arange(coef.shape[0]) // (hdr['ri'] * nb)
    for c in range(len(hdr['comps'])):
        sel = np.nonzero(blk_comp == c)[0]
        d = coef[sel, 0]
        cs = np.cumsum(d)
        seg = interval[sel]
        first = np.r_[True, seg[1:] != seg[:-1]]
        head = np.maximum.accumulate(np.where(first, np.arange(len(sel)), 0))
        coef[sel, 0] = cs - (cs - d)[head]


def subsequences(hdr, buf, starts, S):
    """[(interval, Bits, start bit, end bit, first of its interval)]: each interval cut into S-bit pieces (at least one)"""
    ends = list(starts[1:hdr['n_intervals']]) + [len(buf)]
    subs = []
    for i in range(hdr['n_intervals']):
        lo = min(starts[i], len(buf)) if i < len(starts) else len(buf)
        hi = max(lo, min(ends[i], len(buf)) if i < len(ends) else len(buf))
        nbits, bits = 8 * (hi - lo), Bits(buf, lo, hi)
        for j in range(max(1, -(-nbits // S))):
            subs.append((i, bits, j * S, min((j + 1) * S, nbits), j == 0))
    return subs


def self_sync(hdr, buf, starts, S, max_rounds):
    """The GPU's entropy decode.  Round 0 decodes every subsequence from (its first bit, block 0, k 0) and records its
    exit; each further round sets start_j := exit_{j-1} and re-decodes the subsequences whose start changed.  At the
    fixed point every start is exact by induction from the first subsequence of each interval.  After max_rounds rounds
    a serial pass per interval re-decodes each subsequence whose start still differs from its predecessor's exit
    (max_rounds 0: every subsequence).  The write pass then decodes each subsequence again from its settled start into
    block (interval base + the block starts of the subsequences before it).
    -> (coefficients like coefficients_serial, rounds that decoded something, fallback decodes)"""
    nb = len(hdr['blocks'])
    subs = subsequences(hdr, buf, starts, S)
    n = len(subs)
    start = [(s[2], 0, 0) for s in subs]
    exit_, count = [None] * n, [0] * n
    rounds = 0
    for r in range(max_rounds):
        prev = list(exit_)
        work = False
        for j in range(n):
            if r > 0:
                if subs[j][4] or prev[j - 1] == start[j]:
                    continue
                start[j] = prev[j - 1]
            exit_[j], count[j] = decode_run(hdr, subs[j][1], start[j], subs[j][3])
            work = True
        rounds += work
        if not work:
            break
    fallbacks = 0
    for j in range(n):
        if max_rounds == 0 or (not subs[j][4] and exit_[j - 1] != start[j]):
            if not subs[j][4]:
                start[j] = exit_[j - 1]
            exit_[j], count[j] = decode_run(hdr, subs[j][1], start[j], subs[j][3])
            fallbacks += 1
    coef = np.zeros((hdr['mx'] * hdr['my'] * nb, 64), dtype=np.int64)
    acc = 0
    for j in range(n):
        i = subs[j][0]
        acc = 0 if subs[j][4] else acc
        base, cnt = i * hdr['ri'] * nb, interval_blocks(hdr, i)

        def emit(b, z, v, at=base + acc, lim=cnt - acc):
            if b < lim:                            # b == -1: the block the previous subsequence began
                coef[at + b, z] = v
        decode_run(hdr, subs[j][1], start[j], subs[j][3], emit, max_blocks=max(cnt - acc, 0))
        acc += count[j]
    resolve_dc(hdr, coef)
    return coef, rounds, fallbacks


# ---------------------------------------------------------------------------------------------------- reconstruction
FIX = dict(p298=2446, p390=3196, p541=4433, p765=6270, p899=7373, p1175=9633, p1501=12299, p1847=15137, p1961=16069,
           p2053=16819, p2562=20995, p3072=25172)
CONST_BITS, PASS1_BITS = 13, 2


def _idct_1d(s0, s1, s2, s3, s4, s5, s6, s7, shift):
    F = FIX
    z1 = (s2 + s6) * F['p541']
    tmp2 = z1 + s6 * -F['p1847']
    tmp3 = z1 + s2 * F['p765']
    tmp0 = (s0 + s4) << CONST_BITS
    tmp1 = (s0 - s4) << CONST_BITS
    tmp10, tmp13, tmp11, tmp12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    t0, t1, t2, t3 = s7, s5, s3, s1
    z1, z2, z3, z4 = t0 + t3, t1 + t2, t0 + t2, t1 + t3
    z5 = (z3 + z4) * F['p1175']
    t0, t1, t2, t3 = t0 * F['p298'], t1 * F['p2053'], t2 * F['p3072'], t3 * F['p1501']
    z1, z2, z3, z4 = z1 * -F['p899'], z2 * -F['p2562'], z3 * -F['p1961'], z4 * -F['p390']
    z3 = z3 + z5
    z4 = z4 + z5
    t0, t1, t2, t3 = t0 + z1 + z3, t1 + z2 + z4, t2 + z2 + z3, t3 + z1 + z4
    r = 1 << (shift - 1)
    return [(tmp10 + t3 + r) >> shift, (tmp11 + t2 + r) >> shift, (tmp12 + t1 + r) >> shift,
            (tmp13 + t0 + r) >> shift, (tmp13 - t0 + r) >> shift, (tmp12 - t1 + r) >> shift,
            (tmp11 - t2 + r) >> shift, (tmp10 - t3 + r) >> shift]


def idct_islow(coef, q):
    """coef int64 [N, 64] natural order, q [64] -> uint8 [N, 8, 8] (jidctint.c, range-limited like IDCT_range_limit)"""
    d = (coef * q[None, :]).reshape(-1, 8, 8)
    cols = _idct_1d(*[d[:, i, :] for i in range(8)], CONST_BITS - PASS1_BITS)      # pass 1: columns
    ws = np.stack(cols, axis=1)                                                    # [N, row, col]
    rows = _idct_1d(*[ws[:, :, i] for i in range(8)], CONST_BITS + PASS1_BITS + 3)  # pass 2: rows
    out = np.stack(rows, axis=2)
    m = out & 1023
    s = np.where(m >= 512, m - 1024, m)
    return np.clip(s + 128, 0, 255).astype(np.uint8)


def planes(hdr, coef):
    """component planes, padded to the MCU grid"""
    nb = len(hdr['blocks'])
    out = []
    for ci, c in enumerate(hdr['comps']):
        H, V = c['h'], c['v']
        pl = np.zeros((hdr['my'] * V * 8, hdr['mx'] * H * 8), dtype=np.uint8)
        idx = [bi for bi, b in enumerate(hdr['blocks']) if b[0] == ci]
        px = idct_islow(coef.reshape(-1, nb, 64)[:, idx].reshape(-1, 64), c['q']).reshape(hdr['my'], hdr['mx'], V, H, 8, 8)
        out.append(px.transpose(0, 2, 4, 1, 3, 5).reshape(pl.shape))
    return out


def upsample_h2v1(p, dw):
    """jdsample.c h2v1_fancy_upsample on the first dw (> 2) columns"""
    x = p.astype(np.int32)
    n = max(dw, 2)
    cur = x[:, :n]
    left = np.concatenate([cur[:, :1], cur[:, :-1]], axis=1)
    right = np.concatenate([cur[:, 1:], cur[:, -1:]], axis=1)
    out = np.empty((x.shape[0], 2 * n), dtype=np.int32)
    out[:, 0::2] = (3 * cur + left + 1) >> 2
    out[:, 1::2] = (3 * cur + right + 2) >> 2
    out[:, 0] = cur[:, 0]
    out[:, 2 * dw - 1] = cur[:, dw - 1]
    return out.astype(np.uint8)


def upsample_h2v2(p, dw, dh):
    """jdsample.c h2v2_fancy_upsample on the first dw (> 2) columns: rows above / below replicated at the real
    downsampled height"""
    x = p.astype(np.int32)
    rows = np.arange(x.shape[0])
    above = x[np.clip(rows - 1, 0, max(dh - 1, 0))]
    below = x[np.minimum(rows + 1, dh - 1) if dh > 0 else rows]
    n = max(dw, 2)
    out = np.empty((2 * x.shape[0], 2 * n), dtype=np.int32)
    for v, nb in ((0, above), (1, below)):
        col = 3 * x + nb                                        # colsum
        cur = col[:, :n]
        left = np.concatenate([cur[:, :1], cur[:, :-1]], axis=1)
        right = np.concatenate([cur[:, 1:], cur[:, -1:]], axis=1)
        o = np.empty((x.shape[0], 2 * n), dtype=np.int32)
        o[:, 0::2] = (3 * cur + left + 8) >> 4
        o[:, 1::2] = (3 * cur + right + 7) >> 4
        o[:, 0] = (4 * cur[:, 0] + 8) >> 4
        o[:, 2 * dw - 1] = (4 * cur[:, dw - 1] + 7) >> 4
        out[v::2] = o
    return out.astype(np.uint8)


def ycc_to_rgb(y, cb, cr):
    """jdcolor.c ycc_rgb_convert"""
    x = np.arange(256, dtype=np.int64) - 128
    cr_r = (91881 * x + 32768) >> 16
    cb_b = (116130 * x + 32768) >> 16
    cr_g = -46802 * x
    cb_g = -22554 * x + 32768
    y = y.astype(np.int64)
    r = y + cr_r[cr]
    g = y + ((cb_g[cb] + cr_g[cr]) >> 16)
    b = y + cb_b[cb]
    return np.clip(np.stack([r, g, b], axis=-1), 0, 255).astype(np.uint8)


def reconstruct(hdr, coef):
    w, h = hdr['w'], hdr['h']
    pls = planes(hdr, coef)
    if len(pls) == 1:
        g = pls[0][:h, :w]
        return np.repeat(g[:, :, None], 3, axis=2)
    y = pls[0]
    hmax, vmax = hdr['hmax'], hdr['vmax']
    dw, dh = -(-w // hmax), -(-h // vmax)
    chroma = []
    for p in pls[1:]:
        if dw <= 2:                            # libjpeg-turbo's jinit_upsampler: fancy only when wider than 2
            p = np.repeat(np.repeat(p, hmax, axis=1), vmax, axis=0)
        elif (hmax, vmax) == (2, 1):
            p = upsample_h2v1(p, dw)
        elif (hmax, vmax) == (2, 2):
            p = upsample_h2v2(p, dw, dh)
        chroma.append(p[:h, :w])
    return ycc_to_rgb(y[:h, :w], chroma[0], chroma[1])


def decode(data, S=None, max_rounds=None):
    """np.asarray(PIL.Image.open(data).convert('RGB')) for a 'gpu' stream; serial entropy decode unless S is given"""
    route, hdr = parse(data)
    if route != 'gpu':
        raise JpegError(f'not a GPU stream: {hdr}')
    buf, starts = unstuff(bytes(data), hdr['seg'])
    if S is None:
        coef = coefficients_serial(hdr, buf, starts)
    else:
        coef = self_sync(hdr, buf, starts, S, max_rounds)[0]
    return reconstruct(hdr, coef)
