// libpifpaf_b200 -- baseline JPEG decode on the GPU, bit-identical to Pillow (libjpeg-turbo's defaults).
//
// The reference decodes every file with PIL.Image.open(f).convert('RGB') (datasets/image_list.py:18).  Pillow's
// libjpeg-turbo uses the accurate integer IDCT (jidctint), fancy upsampling (jdsample) and the fixed-point YCbCr->RGB
// tables (jdcolor) by default: integer arithmetic throughout, restated here so the decoded image equals Pillow's.
//
// Host: marker parse: Huffman tables (9-bit lookup + canonical maxcode / valoffset), quantisation tables in natural
// order, the MCU layout, validation; a walk over the scan (SSE2, sixteen bytes a step) for its end and the markers
// inside it, which is also the staging copy of its bytes; the restart-interval table; one pinned copy to the device.
// Damaged streams, as libjpeg decodes them (jdhuff.c, jdmarker.c):
//   - The scan ends at the first marker after the SOS that is not RSTn (or a code below SOF0, which libjpeg's resync
//     skips); FF fill bytes and FF00 are not markers.  Bytes after it (a trailer, a second image) are not staged.
//   - Every marker in the scan ends a data segment.  Interval i > 0 expects RST((i - 1) mod 8) and gets its data
//     segment by jpeg_resync_to_restart: the expected marker or one too far from it is taken, a prior one (or a code
//     below SOF0) is skipped with its data, one of the next two or the scan's end is left unread: an empty segment.
//   - Bits past a segment read as zeros.  The MCU that consumes them is finished from zeros (insufficient_data); the
//     interval's later blocks stay all zero with an absolute DC of 0.  An empty segment after a starved interval
//     decodes nothing (the flag survives a marker left unread); otherwise its first MCU is decoded from zeros.
//   - JFIF needs an APP0 of at least 14 bytes; a JFIF / Adobe segment too short for Pillow's parser takes Pillow's
//     route, which raises as the reference's loader does.
//   - A damaged block can overshoot the IDCT's 16-bit lanes.  The IDCT follows the x86 SIMD code (jidctint-sse2 /
//     -avx2) of the libjpeg-turbo bundled with Pillow's x86-64 wheels, which Pillow runs there: 16-bit products and
//     sums, pass 1's shortcut for blocks whose coefficient rows 1..7 are zero, saturating packs.  Pillow on ARM (NEON),
//     or with JSIMD_FORCENONE, gives other pixels for such blocks; clean streams decode the same on every back end.
// Device, per batch:
//   k_jpeg_unstuff_count / _scan / _write   drop FF fill bytes, the 00 of FF00 and the markers (order-preserving
//                                           compaction), record the compacted start of every data segment
//   k_jpeg_subseq_setup                     cut each interval into SUBSEQ_BITS-bit subsequences
//   k_jpeg_sync (one launch per round)      self-synchronising Huffman decode (Weissenberger & Schmidt, ICPP 2018):
//                                           start_j := exit_{j-1} until no start changes, at most max_rounds rounds
//   k_jpeg_settle                           one warp per interval: serial re-decode of every subsequence whose start
//                                           still differs from its predecessor's exit, then the block prefix sum
//   k_jpeg_write                            decode again from the settled starts, int16 coefficients in natural order
//   k_jpeg_dc                               DC differences -> values: segmented prefix sum per component and interval
//   k_jpeg_idct                             jidctint islow as the x86 SIMD code of Pillow's libjpeg-turbo computes it
//                                           (16-bit products and sums, pass 1's shortcut, saturating packs),
//                                           one thread per block, planes padded to the MCU grid
//   k_jpeg_color                            fancy upsampling (h2v1 / h2v2) + YCbCr->RGB, uint8 HWC
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <vector>
#if defined(__SSE2__)
#include <emmintrin.h>
#endif

#include "common.cuh"

namespace {

constexpr int LOOKUP_BITS = 9;
constexpr int SUBSEQ_BITS = 1024;          // S: bits of entropy-coded data per thread and round
constexpr int DEFAULT_ROUNDS = 16;
constexpr int CHUNK = 256;                 // bytes per thread of the unstuffing pass
constexpr int MAX_BLOCKS_PER_MCU = 6;      // 4:2:0: four luma blocks and two chroma blocks

__constant__ uint8_t c_zigzag[64] = {
    0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21,
    28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61,
    54, 47, 55, 62, 63};
const uint8_t h_zigzag[64] = {
    0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21,
    28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61,
    54, 47, 55, 62, 63};

struct Huff {                              // one DHT table, decode form
    uint16_t lookup[1 << LOOKUP_BITS];     // len << 8 | symbol for codes of <= 9 bits, 0: longer code
    int32_t maxcode[18];                   // largest code of each length (-1: none); [17] sentinel
    int32_t valoffset[17];                 // symbol index = valoffset[len] + code
    uint8_t vals[256];
};

struct Img {                               // one GPU-route image of the batch
    int32_t w, h, ncomp, hmax, vmax, mx, my, bpm, ri, n_int;
    int32_t blk_comp[MAX_BLOCKS_PER_MCU], blk_v[MAX_BLOCKS_PER_MCU], blk_h[MAX_BLOCKS_PER_MCU];
    int32_t comp_h[3], comp_v[3], comp_first[3];   // sampling, first block of the component in an MCU
    int32_t plane_w[3], plane_h[3];
    int64_t plane_off[3];                  // into the plane buffer
    int64_t seg_off;                       // raw scan segment in the byte buffer; its compacted bytes at the same offset
    int32_t seg_len, chunk_base, n_chunks, int_base, sub_base, sub_cap;
    int32_t seg_base, n_seg;               // data segments (one more than the markers in the scan)
    int64_t blk_base, px_base, out_off;    // first coefficient block, first output pixel of the batch, RGB byte offset
    int32_t huff[3][2], quant[3];          // table indices per component (DC, AC)
};

struct Dev {                               // device pointers of one decode
    const Img* img;
    const Huff* huff;
    const int32_t* quant;                  // [n][64] natural order
    const int32_t* chunk_img;
    const uint8_t* raw;
    uint8_t* comp;
    int32_t* chunk_keep;                   // per chunk: kept bytes, then (after the scan) their compacted offset
    int32_t* chunk_rst;
    int32_t* comp_len;                     // per image
    const int32_t* int_seg;                // per interval: its data segment, -1: empty (a marker left unread)
    int32_t* seg_lo;                       // per data segment: compacted start byte
    int32_t* int_lo;                       // per interval: compacted start and end byte
    int32_t* int_hi;
    int32_t* int_blocks;                   // per interval: block starts up to the MCU that ran past its data
    int32_t* int_img;
    int32_t* int_sub;                      // first subsequence, number of subsequences
    int32_t* int_nsub;
    int32_t* sub_int;                      // per subsequence slot: global interval (-1: unused slot)
    int32_t* sub_j;
    long long* start;                      // packed state (bit << 16 | block in MCU << 8 | k); -1: not decoded
    long long* exit0;
    long long* exit1;
    int32_t* count;                        // block starts of the subsequence's decode
    int32_t* acc;                          // block starts of the subsequences before it in its interval
    int16_t* coef;
    uint8_t* plane;
    uint8_t* out;
    unsigned long long* stats;             // [0] rounds that decoded something, [1] fallback decodes
};

__host__ __device__ inline long long pack_state(long long bit, int blk, int k) { return (bit << 16) | (blk << 8) | k; }

// ------------------------------------------------------------------------------------------------ unstuffing
// byte i of a scan is data (1) unless it is an FF fill byte, the 00 of FF00 or a marker's FF (0), or a marker's code
// (2): an FF is data only before 00 (jpeg_fill_bit_buffer)
__device__ __forceinline__ int classify(const uint8_t* s, int i, int n) {
    const uint8_t b = s[i];
    if (b == 0xFF) return i + 1 < n && s[i + 1] == 0x00 ? 1 : 0;
    if (i > 0 && s[i - 1] == 0xFF) return b == 0x00 ? 0 : 2;
    return 1;
}

__global__ void __launch_bounds__(256) k_jpeg_unstuff_count(Dev d, int n_chunks) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= n_chunks) return;
    const Img& im = d.img[d.chunk_img[c]];
    const uint8_t* s = d.raw + im.seg_off;
    const int lo = (c - im.chunk_base) * CHUNK, hi = min(lo + CHUNK, im.seg_len);
    int keep = 0, rst = 0;
    for (int i = lo; i < hi; i++) {
        const int t = classify(s, i, im.seg_len);
        keep += t == 1;
        rst += t == 2;
    }
    d.chunk_keep[c] = keep;
    d.chunk_rst[c] = rst;
}

// exclusive block-wide scan of one value per thread (blockDim.x == 1024); returns the block total in *total
__device__ int block_exclusive_scan(int v, int* total) {
    __shared__ int warp_sums[32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int x = v;
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) warp_sums[warp] = x;
    __syncthreads();
    if (warp == 0) {
        int w = warp_sums[lane];
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, w, o);
            if (lane >= o) w += y;
        }
        warp_sums[lane] = w;
    }
    __syncthreads();
    const int incl = x + (warp > 0 ? warp_sums[warp - 1] : 0);
    *total = warp_sums[31];
    __syncthreads();
    return incl - v;
}

// one CTA per image: chunk offsets (kept bytes, markers), compacted length
__global__ void __launch_bounds__(1024) k_jpeg_unstuff_scan(Dev d) {
    const Img& im = d.img[blockIdx.x];
    int carry_k = 0, carry_r = 0;
    for (int t0 = 0; t0 < im.n_chunks; t0 += 1024) {
        const int c = im.chunk_base + t0 + threadIdx.x;
        const bool ok = t0 + (int)threadIdx.x < im.n_chunks;
        int tk, tr;
        const int ek = block_exclusive_scan(ok ? d.chunk_keep[c] : 0, &tk);
        const int er = block_exclusive_scan(ok ? d.chunk_rst[c] : 0, &tr);
        if (ok) {
            d.chunk_keep[c] = carry_k + ek;
            d.chunk_rst[c] = carry_r + er;
        }
        carry_k += tk;
        carry_r += tr;
    }
    if (threadIdx.x == 0) d.comp_len[blockIdx.x] = carry_k;
    if (threadIdx.x == 0) d.seg_lo[im.seg_base] = 0;
    for (int i = threadIdx.x; i < im.n_int; i += 1024) d.int_img[im.int_base + i] = blockIdx.x;
}

__global__ void __launch_bounds__(256) k_jpeg_unstuff_write(Dev d, int n_chunks) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= n_chunks) return;
    const Img& im = d.img[d.chunk_img[c]];
    const uint8_t* s = d.raw + im.seg_off;
    uint8_t* o = d.comp + im.seg_off;
    const int lo = (c - im.chunk_base) * CHUNK, hi = min(lo + CHUNK, im.seg_len);
    int out = d.chunk_keep[c], rst = d.chunk_rst[c];
    for (int i = lo; i < hi; i++) {
        const int t = classify(s, i, im.seg_len);
        if (t == 1) {
            o[out++] = s[i];
        } else if (t == 2) {
            if (++rst < im.n_seg) d.seg_lo[im.seg_base + rst] = out;
        }
    }
}

// one CTA per image: interval bounds, subsequence slots (S bits each, at least one per interval)
__global__ void __launch_bounds__(1024) k_jpeg_subseq_setup(Dev d) {
    const Img& im = d.img[blockIdx.x];
    const int len = d.comp_len[blockIdx.x];
    int carry = 0;
    for (int t0 = 0; t0 < im.n_int; t0 += 1024) {
        const int i = t0 + threadIdx.x;
        const bool ok = i < im.n_int;
        int lo = 0, hi = 0, nsub = 0;
        if (ok) {
            const int sg = d.int_seg[im.int_base + i];
            if (sg >= 0) {
                lo = min(d.seg_lo[im.seg_base + sg], len);
                hi = max(lo, sg + 1 < im.n_seg ? min(d.seg_lo[im.seg_base + sg + 1], len) : len);
            }
            nsub = max(1, (int)(((long long)(hi - lo) * 8 + SUBSEQ_BITS - 1) / SUBSEQ_BITS));
        }
        int total;
        const int first = carry + block_exclusive_scan(nsub, &total);
        if (ok) {
            d.int_lo[im.int_base + i] = lo;
            d.int_hi[im.int_base + i] = hi;
            d.int_sub[im.int_base + i] = im.sub_base + first;
            d.int_nsub[im.int_base + i] = nsub;
        }
        carry += total;
    }
    __syncthreads();
    // fill the slots: interval of each (a binary search over the interval table), unused slots -1
    for (int j = threadIdx.x; j < im.sub_cap; j += 1024) {
        const int g = im.sub_base + j;
        int sel = -1, jj = 0;
        if (j < carry) {
            int a = 0, b = im.n_int - 1;
            while (a < b) {
                const int m = (a + b + 1) >> 1;
                if (d.int_sub[im.int_base + m] <= g) a = m; else b = m - 1;
            }
            sel = im.int_base + a;
            jj = g - d.int_sub[sel];
        }
        d.sub_int[g] = sel;
        d.sub_j[g] = jj;
        d.start[g] = -1;
        d.count[g] = 0;
    }
}

// ------------------------------------------------------------------------------------------------ Huffman decoding
struct BitReader {
    const uint8_t* p;                      // the interval's compacted bytes
    int n;                                 // its length: bits past the end read as zeros (libjpeg at a marker)
    __device__ __forceinline__ unsigned peek24(long long pos) const {
        const long long i = pos >> 3;
        unsigned v = 0;
#pragma unroll
        for (int k = 0; k < 4; k++) v = (v << 8) | (i + k < n ? (unsigned)__ldg(p + i + k) : 0u);
        return v << (pos & 7);             // the next 24+ bits, MSB first
    }
    __device__ __forceinline__ int bits(long long pos, int cnt) const { return cnt ? (int)(peek24(pos) >> (32 - cnt)) : 0; }
};

__device__ __forceinline__ int huff_decode(const Huff& t, const BitReader& br, long long pos, int* len) {
    const unsigned w = br.peek24(pos);
    const int e = t.lookup[w >> (32 - LOOKUP_BITS)];
    if (e) {
        *len = e >> 8;
        return e & 255;
    }
    int l = LOOKUP_BITS + 1;
    int code = (int)(w >> (32 - l));
    while (l <= 16 && code > t.maxcode[l]) {
        l++;
        code = (int)(w >> (32 - l));
    }
    if (l > 16) {                          // no such code: 17 bits read and a zero symbol, like libjpeg
        *len = 17;
        return 0;
    }
    *len = l;
    return t.vals[(t.valoffset[l] + code) & 255];
}

__device__ __forceinline__ int extend(int v, int s) { return (s && v < (1 << (s - 1))) ? v - (1 << s) + 1 : v; }

// Decode from state until the first codeword boundary at or after end_bit; with coef, also write the coefficients
// (DC: its difference) of block base + (block starts so far - 1) while that is below limit, and stop before the DC
// of block `limit`.  The tail of an interval (end_bit: its last bit) goes on to the end of an MCU whose bits run past
// the data, and decodes one more MCU when the data ends exactly at an MCU boundary: libjpeg finishes the MCU that runs
// out of data from zero bits.  Returns the exit state; *nstart = block starts.
template <bool WRITE>
__device__ long long decode_run(const Dev& d, const Img& im, const BitReader& br, long long state, long long end_bit,
                                bool tail, int* nstart, int16_t* coef = nullptr, int limit = 0) {
    long long pos = state >> 16;
    int blk = (int)((state >> 8) & 255), k = (int)(state & 255);
    int ns = 0;
    while (pos < end_bit || (tail && (pos == end_bit || blk != 0 || k != 0))) {
        const int c = im.blk_comp[blk];
        if (k == 0) {
            if (WRITE && ns >= limit) break;
            int len;
            const int s = huff_decode(d.huff[im.huff[c][0]], br, pos, &len);
            pos += len;
            const int v = extend(br.bits(pos, s), s);
            pos += s;
            ns++;
            if (WRITE) coef[(long long)(ns - 1) * 64] = (int16_t)v;
            k = 1;
        } else {
            int len;
            const int rs = huff_decode(d.huff[im.huff[c][1]], br, pos, &len);
            pos += len;
            const int r = rs >> 4, s = rs & 15;
            if (s) {
                k += r;
                const int v = extend(br.bits(pos, s), s);
                pos += s;
                if (WRITE && ns - 1 < limit) coef[(long long)(ns - 1) * 64 + c_zigzag[min(k, 63)]] = (int16_t)v;
                k++;
            } else if (r == 15) {
                k += 16;
            } else {
                k = 64;
            }
        }
        if (k >= 64) {
            k = 0;
            blk = blk + 1 == im.bpm ? 0 : blk + 1;
        }
    }
    *nstart = ns;
    return pack_state(pos, blk, k);
}

struct SubView {
    const Img* im;
    BitReader br;
    long long end_bit;
    bool first, last;
};

__device__ __forceinline__ SubView sub_view(const Dev& d, int g) {
    const int iv = d.sub_int[g], j = d.sub_j[g];
    const int lo = d.int_lo[iv], hi = d.int_hi[iv];
    SubView v;
    v.im = &d.img[d.int_img[iv]];
    v.br.p = d.comp + v.im->seg_off + lo;
    v.br.n = hi - lo;
    v.end_bit = min((long long)(j + 1) * SUBSEQ_BITS, (long long)(hi - lo) * 8);
    v.first = j == 0;
    v.last = j + 1 == d.int_nsub[iv];
    return v;
}

// round 0: every subsequence from (its first bit, block 0, k 0); round r: start := the predecessor's exit of round
// r - 1, re-decoded only where that changed the start.  exits ping-pong between rounds.
__global__ void __launch_bounds__(128) k_jpeg_sync(Dev d, int n_slots, int round) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= n_slots || d.sub_int[g] < 0) return;
    const long long* prev = round & 1 ? d.exit0 : d.exit1;
    long long* cur = round & 1 ? d.exit1 : d.exit0;
    const SubView v = sub_view(d, g);
    long long st;
    if (round == 0) {
        st = pack_state((long long)d.sub_j[g] * SUBSEQ_BITS, 0, 0);
    } else {
        st = v.first ? d.start[g] : prev[g - 1];
        if (st == d.start[g]) {
            cur[g] = prev[g];
            return;
        }
    }
    int ns;
    cur[g] = decode_run<false>(d, *v.im, v.br, st, v.end_bit, v.last, &ns);
    d.start[g] = st;
    d.count[g] = ns;
    atomicMax(&d.stats[0], (unsigned long long)(round + 1));
}

// one warp per interval: re-decode, in order, every subsequence whose start is not its predecessor's exit (all of
// them without a sync round), then the exclusive prefix of the block starts
__global__ void __launch_bounds__(128) k_jpeg_settle(Dev d, int n_int_total, int final_buf) {
    const int iv = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (iv >= n_int_total) return;
    volatile long long* ex = final_buf ? d.exit1 : d.exit0;     // written by one lane, read by the next
    const int s0 = d.int_sub[iv], ns = d.int_nsub[iv];
    int carry = 0;
    unsigned long long fallbacks = 0;
    for (int t0 = 0; t0 < ns; t0 += 32) {
        const int g = s0 + t0 + lane;
        const bool ok = t0 + lane < ns;
        for (;;) {
            bool bad = false;
            if (ok) {
                const long long want = t0 + lane == 0 ? pack_state(0, 0, 0) : ex[g - 1];
                bad = d.start[g] != want;
            }
            const unsigned m = __ballot_sync(0xffffffffu, bad);
            if (!m) break;
            const int L = __ffs(m) - 1;
            if (lane == L) {
                const SubView v = sub_view(d, g);
                const long long st = t0 + lane == 0 ? pack_state(0, 0, 0) : ex[g - 1];
                int n;
                ex[g] = decode_run<false>(d, *v.im, v.br, st, v.end_bit, v.last, &n);
                d.start[g] = st;
                d.count[g] = n;
                fallbacks++;
            }
            __syncwarp();
        }
        int x = ok ? d.count[g] : 0;
        const int own = x;
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, x, o);
            if (lane >= o) x += y;
        }
        if (ok) d.acc[g] = carry + x - own;
        carry += __shfl_sync(0xffffffffu, x, 31);
    }
    const unsigned long long warp_fallbacks = __reduce_add_sync(0xffffffffu, (unsigned)fallbacks);   // every lane's
    if (lane == 0 && warp_fallbacks) atomicAdd(&d.stats[1], warp_fallbacks);
    if (lane == 0) d.int_blocks[iv] = carry;
}

__device__ __forceinline__ int interval_block_count(const Img& im, int local) {
    const long long mcu0 = (long long)local * im.ri;
    return (int)((min(mcu0 + im.ri, (long long)im.mx * im.my) - mcu0) * im.bpm);
}

// blocks of an interval the decode keeps: those started up to the MCU that ran past its data.  An empty interval
// after a starved one (all its blocks started there, or itself empty) keeps none.
__device__ __forceinline__ int interval_live(const Dev& d, const Img& im, int local) {
    const int iv = im.int_base + local;
    if (local > 0 && d.int_seg[iv] < 0 &&
        (d.int_seg[iv - 1] < 0 || d.int_blocks[iv - 1] <= interval_block_count(im, local - 1)))
        return 0;
    return min(d.int_blocks[iv], interval_block_count(im, local));
}

// ------------------------------------------------------------------------------------------------ write pass
__global__ void __launch_bounds__(128) k_jpeg_write(Dev d, int n_slots) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= n_slots || d.sub_int[g] < 0) return;
    const int iv = d.sub_int[g];
    const SubView v = sub_view(d, g);
    const Img& im = *v.im;
    const int local = iv - im.int_base;
    const long long mcu0 = (long long)local * im.ri;
    const int cnt = interval_live(d, im, local);
    const int acc = d.acc[g];
    const long long st = d.start[g];
    const int mid = (st & 255) != 0;       // the first block was begun by the previous subsequence
    if (acc - mid >= cnt) return;
    int16_t* base = d.coef + (im.blk_base + mcu0 * im.bpm + acc) * 64;
    int ns;
    decode_run<true>(d, im, v.br, st, v.end_bit, v.last, &ns, base, cnt - acc);
}

// DC differences -> values: one CTA per (image, component), prefix sum over the component's blocks in scan order,
// restarted at every interval; a block past its interval's live blocks keeps an absolute DC of 0
__global__ void __launch_bounds__(1024) k_jpeg_dc(Dev d) {
    const Img& im = d.img[blockIdx.x / 3];
    const int c = blockIdx.x % 3;
    if (c >= im.ncomp) return;
    const int nbc = im.comp_h[c] * im.comp_v[c];
    const long long n = (long long)im.mx * im.my * nbc;
    __shared__ int sv[1024];
    __shared__ unsigned char sf[1024];
    int carry = 0;
    for (long long t0 = 0; t0 < n; t0 += 1024) {
        const long long e = t0 + threadIdx.x;
        const bool ok = e < n;
        long long blk = 0;
        int v = 0, f = 1;
        if (ok) {
            const long long mcu = e / nbc;
            const int t = (int)(e % nbc);
            blk = im.blk_base + mcu * im.bpm + im.comp_first[c] + t;
            const int local = (int)(mcu / im.ri);
            const bool dead = (mcu - (long long)local * im.ri) * im.bpm + im.comp_first[c] + t >= interval_live(d, im, local);
            v = dead ? 0 : d.coef[blk * 64];
            f = (t == 0 && mcu % im.ri == 0) || dead;
        }
        sv[threadIdx.x] = v;
        sf[threadIdx.x] = (unsigned char)f;
        __syncthreads();
        for (int o = 1; o < 1024; o <<= 1) {              // segmented inclusive scan (Hillis-Steele)
            int x = sv[threadIdx.x];
            unsigned char fl = sf[threadIdx.x];
            if (threadIdx.x >= o && !fl) {
                x += sv[threadIdx.x - o];
                fl = sf[threadIdx.x - o];
            }
            __syncthreads();
            sv[threadIdx.x] = x;
            sf[threadIdx.x] = fl;
            __syncthreads();
        }
        const int val = sv[threadIdx.x] + (sf[threadIdx.x] ? 0 : carry);
        if (ok) d.coef[blk * 64] = (int16_t)val;          // libjpeg: (JCOEF) of the int predictor
        __syncthreads();
        if (threadIdx.x == 1023) sv[0] = val;
        __syncthreads();
        carry = sv[0];
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------------ reconstruction
constexpr int CONST_BITS = 13, PASS1_BITS = 2;

// jidctint's 1-D pass as libjpeg-turbo's SSE2 / AVX2 code computes it: in0 +- in4, in7 + in3 and in5 + in1 are 16-bit
// adds (paddw / psubw); every other term is a pmaddwd of 16-bit inputs into 32 bits, which does not overflow
__device__ __forceinline__ long long add16(long long a, long long b) { return (int16_t)(a + b); }

__device__ __forceinline__ void idct_1d(const int* s, int stride, int shift, int* out, int ostride) {
    const long long s0 = s[0], s1 = s[stride], s2 = s[2 * stride], s3 = s[3 * stride], s4 = s[4 * stride],
                    s5 = s[5 * stride], s6 = s[6 * stride], s7 = s[7 * stride];
    long long z1 = (s2 + s6) * 4433;
    const long long tmp2 = z1 + s6 * -15137, tmp3 = z1 + s2 * 6270;
    const long long tmp0 = add16(s0, s4) * (1 << CONST_BITS), tmp1 = add16(s0, -s4) * (1 << CONST_BITS);
    const long long tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
    long long t0 = s7, t1 = s5, t2 = s3, t3 = s1;
    z1 = t0 + t3;
    long long z2 = t1 + t2, z3 = add16(t0, t2), z4 = add16(t1, t3);
    const long long z5 = (z3 + z4) * 9633;
    t0 *= 2446; t1 *= 16819; t2 *= 25172; t3 *= 12299;
    z1 *= -7373; z2 *= -20995; z3 *= -16069; z4 *= -3196;
    z3 += z5; z4 += z5;
    t0 += z1 + z3; t1 += z2 + z4; t2 += z2 + z3; t3 += z1 + z4;
    const long long r = 1LL << (shift - 1);
    out[0 * ostride] = (int)((tmp10 + t3 + r) >> shift);
    out[7 * ostride] = (int)((tmp10 - t3 + r) >> shift);
    out[1 * ostride] = (int)((tmp11 + t2 + r) >> shift);
    out[6 * ostride] = (int)((tmp11 - t2 + r) >> shift);
    out[2 * ostride] = (int)((tmp12 + t1 + r) >> shift);
    out[5 * ostride] = (int)((tmp12 - t1 + r) >> shift);
    out[3 * ostride] = (int)((tmp13 + t0 + r) >> shift);
    out[4 * ostride] = (int)((tmp13 - t0 + r) >> shift);
}

__device__ __forceinline__ int find_image(const Img* img, int n, long long v, bool by_pixel) {
    int a = 0, b = n - 1;
    while (a < b) {
        const int m = (a + b + 1) >> 1;
        if ((by_pixel ? img[m].px_base : img[m].blk_base) <= v) a = m; else b = m - 1;
    }
    return a;
}

__global__ void __launch_bounds__(128) k_jpeg_idct(Dev d, int n_img, long long n_blocks) {
    const long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= n_blocks) return;
    const Img& im = d.img[find_image(d.img, n_img, b, false)];
    const long long local = b - im.blk_base;
    const long long mcu = local / im.bpm;
    const int t = (int)(local % im.bpm);
    const int c = im.blk_comp[t];
    const int* q = d.quant + im.quant[c] * 64;
    const int16_t* in = d.coef + b * 64;
    int x[64], ws[64];
    bool rows0 = true;                                     // coefficient rows 1..7 all zero
#pragma unroll
    for (int i = 0; i < 64; i++) {
        x[i] = (int16_t)((int)in[i] * q[i]);              // libjpeg-turbo's SIMD IDCT: pmullw
        if (i >= 8) rows0 = rows0 && in[i] == 0;
    }
    if (rows0) {                                           // pass 1's shortcut: psllw, wrapping in 16 bits
#pragma unroll
        for (int i = 0; i < 64; i++) ws[i] = (int16_t)(x[i & 7] * (1 << PASS1_BITS));
    } else {
#pragma unroll
        for (int col = 0; col < 8; col++) idct_1d(x + col, 8, CONST_BITS - PASS1_BITS, ws + col, 8);
#pragma unroll
        for (int i = 0; i < 64; i++) ws[i] = min(max(ws[i], -32768), 32767);  // packssdw
    }
    const int my = (int)(mcu / im.mx), mx = (int)(mcu % im.mx);
    const int prow = (my * im.comp_v[c] + im.blk_v[t]) * 8, pcol = (mx * im.comp_h[c] + im.blk_h[t]) * 8;
    uint8_t* o = d.plane + im.plane_off[c] + (long long)prow * im.plane_w[c] + pcol;
#pragma unroll
    for (int row = 0; row < 8; row++) {
        int v[8];
        idct_1d(ws + row * 8, 1, CONST_BITS + PASS1_BITS + 3, v, 1);
#pragma unroll
        for (int i = 0; i < 8; i++)                        // packsswb, + 128
            o[(long long)row * im.plane_w[c] + i] = (uint8_t)(min(max(v[i], -128), 127) + 128);
    }
}

// chroma sample at output pixel (x, y): jdsample.c's fancy upsamplers (h2v1, h2v2) on the real downsampled width and
// height; plain replication when that width is 2 or less (jinit_upsampler), and for 4:4:4 the sample itself
__device__ __forceinline__ int chroma(const uint8_t* p, int pw, int hmax, int vmax, int dw, int dh, int x, int y) {
    if (hmax == 1) return p[(long long)y * pw + x];
    const int cx = x >> 1, cy = vmax == 2 ? y >> 1 : y;
    const uint8_t* row = p + (long long)cy * pw;
    if (dw <= 2) return row[cx];
    if (vmax == 1) {
        const int c3 = 3 * row[cx];
        if (x & 1) return cx == dw - 1 ? row[cx] : (c3 + row[cx + 1] + 2) >> 2;
        return cx == 0 ? row[cx] : (c3 + row[cx - 1] + 1) >> 2;
    }
    const int ny = (y & 1) ? min(cy + 1, dh - 1) : max(cy - 1, 0);
    const uint8_t* nrow = p + (long long)ny * pw;
    const int cs = 3 * row[cx] + nrow[cx];
    if (x & 1) return cx == dw - 1 ? (4 * cs + 7) >> 4 : (3 * cs + 3 * row[cx + 1] + nrow[cx + 1] + 7) >> 4;
    return cx == 0 ? (4 * cs + 8) >> 4 : (3 * cs + 3 * row[cx - 1] + nrow[cx - 1] + 8) >> 4;
}

__global__ void __launch_bounds__(256) k_jpeg_color(Dev d, int n_img, long long n_px) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_px) return;
    const Img& im = d.img[find_image(d.img, n_img, t, true)];
    const long long local = t - im.px_base;
    const int y = (int)(local / im.w), x = (int)(local % im.w);
    uint8_t* o = d.out + im.out_off + local * 3;
    const int Y = d.plane[im.plane_off[0] + (long long)y * im.plane_w[0] + x];
    if (im.ncomp == 1) {
        o[0] = o[1] = o[2] = (uint8_t)Y;
        return;
    }
    const int dw = (im.w + im.hmax - 1) / im.hmax, dh = (im.h + im.vmax - 1) / im.vmax;
    const int cb = chroma(d.plane + im.plane_off[1], im.plane_w[1], im.hmax, im.vmax, dw, dh, x, y) - 128;
    const int cr = chroma(d.plane + im.plane_off[2], im.plane_w[2], im.hmax, im.vmax, dw, dh, x, y) - 128;
    const int r = Y + ((91881 * cr + 32768) >> 16);                       // jdcolor.c, SCALEBITS 16
    const int g = Y + ((-22554 * cb + 32768 - 46802 * cr) >> 16);
    const int b = Y + ((116130 * cb + 32768) >> 16);
    o[0] = (uint8_t)min(max(r, 0), 255);
    o[1] = (uint8_t)min(max(g, 0), 255);
    o[2] = (uint8_t)min(max(b, 0), 255);
}

// ------------------------------------------------------------------------------------------------ host: parsing
struct Comp { int id, h, v, tq, td, ta; };
struct Parsed {
    int route;                             // PIFPAF_JPEG_GPU / PIFPAF_JPEG_PILLOW
    int w, h;
    std::vector<Comp> comps;               // in scan order
    int ri;
    int64_t seg_lo, seg_hi;
    std::vector<uint8_t> markers;          // codes of the markers inside the scan, in order
    const Huff* dc[4];
    const Huff* ac[4];
    const int32_t* q[4];
};

int build_huff(const uint8_t* bits, const uint8_t* vals, int n, bool is_dc, Huff* t) {
    std::memset(t, 0, sizeof(Huff));
    int code = 0, p = 0;
    for (int l = 0; l < 18; l++) t->maxcode[l] = -1;
    for (int l = 1; l <= 16; l++) {
        const int cnt = bits[l - 1];
        if (cnt) {
            t->valoffset[l] = p - code;
            for (int i = 0; i < cnt; i++, code++, p++) {
                // jpeg_make_d_derived_tbl: every code fits its length and none is all ones
                if (code + 1 >= (1 << l)) return PIFPAF_E_BADARG;
                if (l <= LOOKUP_BITS) {
                    const int lo = code << (LOOKUP_BITS - l);
                    for (int k = 0; k < (1 << (LOOKUP_BITS - l)); k++) t->lookup[lo + k] = (uint16_t)((l << 8) | vals[p]);
                }
            }
            t->maxcode[l] = code - 1;
        }
        code <<= 1;
    }
    t->maxcode[17] = 0xFFFFF;
    for (int i = 0; i < n; i++) {
        if (is_dc && vals[i] > 15) return PIFPAF_E_BADARG;
        t->vals[i] = vals[i];
    }
    return PIFPAF_OK;
}

// First i' >= i with s[i'] == FF and s[i' + 1] != 00 (a marker or an FF fill byte; n if none), sixteen bytes at a
// time.  With dst, s[i, i') is copied to dst[i - base, ...) on the way (up to 16 bytes more; dst_room bounds it).
// The entropy-coded bytes are read once: the walk is the staging copy.
int64_t find_marker(const uint8_t* s, int64_t i, int64_t n, uint8_t* dst = nullptr, int64_t base = 0,
                    int64_t dst_room = 0) {
#if defined(__SSE2__)
    const __m128i ff = _mm_set1_epi8((char)0xFF), z = _mm_setzero_si128();
    for (; i + 17 <= n; i += 16) {
        const __m128i a = _mm_loadu_si128(reinterpret_cast<const __m128i*>(s + i));
        const __m128i b = _mm_loadu_si128(reinterpret_cast<const __m128i*>(s + i + 1));
        if (dst && i - base + 16 <= dst_room) _mm_storeu_si128(reinterpret_cast<__m128i*>(dst + (i - base)), a);
        const int m = _mm_movemask_epi8(_mm_andnot_si128(_mm_cmpeq_epi8(b, z), _mm_cmpeq_epi8(a, ff)));
        if (m) return i + __builtin_ctz(m);
    }
#endif
    for (; i + 1 < n; i++) {
        if (dst && i - base < dst_room) dst[i - base] = s[i];
        if (s[i] == 0xFF && s[i + 1] != 0) return i;
    }
    return n;
}

#define JPEG_BAD(idx, msg)                                                  \
    do {                                                                    \
        ::pifpaf::set_error("bad argument: JPEG %d: %s", (idx), (msg));     \
        return PIFPAF_E_BADARG;                                             \
    } while (0)

// The tables of one stream live in `tabs` / `quant` (per stream: 4 DC + 4 AC tables, 4 quantisation tables).  A GPU
// route stream's scan bytes are copied to dst (room: the staging bytes left) by the walk that finds the scan's end.
int parse_jpeg(int idx, const uint8_t* s, int64_t n, int64_t max_pixels, Huff* tabs, int32_t* quant, uint8_t* dst,
               int64_t room, Parsed* out) {
    bool have_dc[4] = {}, have_ac[4] = {}, have_q[4] = {};
    bool frame = false, jfif = false;
    int adobe = -1, prec = 0, ri = 0;
    std::vector<Comp> comps;
    out->route = PIFPAF_JPEG_GPU;
    if (n < 4 || s[0] != 0xFF || s[1] != 0xD8) JPEG_BAD(idx, "no SOI marker");
    int64_t pos = 2;
    for (;;) {
        if (pos >= n || s[pos] != 0xFF) JPEG_BAD(idx, "marker expected");
        while (pos < n && s[pos] == 0xFF) pos++;
        if (pos >= n) JPEG_BAD(idx, "truncated marker");
        const int m = s[pos++];
        if (m == 0xD9) JPEG_BAD(idx, "EOI before the scan");
        if ((m >= 0xD0 && m <= 0xD7) || m == 0x01) continue;
        if (pos + 2 > n) JPEG_BAD(idx, "truncated segment length");
        const int64_t ln = (s[pos] << 8) | s[pos + 1];
        if (ln < 2 || pos + ln > n) JPEG_BAD(idx, "segment runs past the end of the stream");
        const uint8_t* seg = s + pos + 2;
        const int64_t sl = ln - 2;
        pos += ln;
        if (m == 0xC0 || m == 0xC1) {
            if (frame) JPEG_BAD(idx, "second frame header");
            if (sl < 6) JPEG_BAD(idx, "short SOF");
            prec = seg[0];
            out->h = (seg[1] << 8) | seg[2];
            out->w = (seg[3] << 8) | seg[4];
            const int nf = seg[5];
            if (sl != 6 + 3 * nf) JPEG_BAD(idx, "bad SOF length");
            for (int i = 0; i < nf; i++) comps.push_back({seg[6 + 3 * i], seg[7 + 3 * i] >> 4, seg[7 + 3 * i] & 15, seg[8 + 3 * i], 0, 0});
            frame = true;
        } else if (m >= 0xC2 && m <= 0xCF && m != 0xC4 && m != 0xC8) {
            out->route = PIFPAF_JPEG_PILLOW;   // progressive, lossless, hierarchical or arithmetic-coded
            return PIFPAF_OK;
        } else if (m == 0xC4) {
            for (int64_t i = 0; i < sl;) {
                if (i + 17 > sl) JPEG_BAD(idx, "short DHT");
                const int tc = seg[i] >> 4, th = seg[i] & 15;
                int cnt = 0;
                for (int k = 1; k <= 16; k++) cnt += seg[i + k];
                if (tc > 1 || th > 3 || cnt > 256 || i + 17 + cnt > sl) JPEG_BAD(idx, "bad DHT");
                if (build_huff(seg + i + 1, seg + i + 17, cnt, tc == 0, tabs + (tc ? 4 : 0) + th) != PIFPAF_OK)
                    JPEG_BAD(idx, "bad Huffman table");
                (tc ? have_ac : have_dc)[th] = true;
                i += 17 + cnt;
            }
        } else if (m == 0xDB) {
            for (int64_t i = 0; i < sl;) {
                const int pq = seg[i] >> 4, tq = seg[i] & 15;
                const int sz = pq ? 128 : 64;
                if (pq > 1 || tq > 3 || i + 1 + sz > sl) JPEG_BAD(idx, "bad DQT");
                for (int k = 0; k < 64; k++)
                    quant[tq * 64 + h_zigzag[k]] = pq ? (seg[i + 1 + 2 * k] << 8) | seg[i + 2 + 2 * k] : seg[i + 1 + k];
                have_q[tq] = true;
                i += 1 + sz;
            }
        } else if (m == 0xDD) {
            if (sl != 2) JPEG_BAD(idx, "bad DRI length");
            ri = (seg[0] << 8) | seg[1];
        } else if (m == 0xE0 || m == 0xEE) {
            // Pillow's parser reads a 16-bit version at byte 5 of a JFIF or Adobe segment and refuses a shorter one
            const bool jf = m == 0xE0 && sl >= 4 && std::memcmp(seg, "JFIF", 4) == 0;
            const bool ad = m == 0xEE && sl >= 5 && std::memcmp(seg, "Adobe", 5) == 0;
            if ((jf || ad) && sl < 7) {
                out->route = PIFPAF_JPEG_PILLOW;
                return PIFPAF_OK;
            }
            jfif = jfif || (jf && sl >= 14 && seg[4] == 0);          // libjpeg's examine_app0: APP0_DATA_LEN
            if (ad && sl >= 12) adobe = seg[11];
        } else if (m == 0xDA) {
            if (!frame) JPEG_BAD(idx, "SOS before SOF");
            if (sl < 1 || sl != 4 + 2 * seg[0]) JPEG_BAD(idx, "bad SOS length");
            const int ns = seg[0], nf = (int)comps.size();
            if (prec != 8 || (nf != 1 && nf != 3)) {
                out->route = PIFPAF_JPEG_PILLOW;
                return PIFPAF_OK;
            }
            if (nf == 3) {
                const bool rgb_ids = comps[0].id == 82 && comps[1].id == 71 && comps[2].id == 66;
                const bool sub_ok = comps[1].h == 1 && comps[1].v == 1 && comps[2].h == 1 && comps[2].v == 1 &&
                                    ((comps[0].h == 1 && comps[0].v == 1) || (comps[0].h == 2 && comps[0].v <= 2 && comps[0].v >= 1));
                if ((adobe >= 0 && adobe != 1) || (!jfif && adobe < 0 && rgb_ids) || !sub_ok) {
                    out->route = PIFPAF_JPEG_PILLOW;
                    return PIFPAF_OK;
                }
            }
            if (ns != nf) {
                out->route = PIFPAF_JPEG_PILLOW;   // one component per scan: a multi-scan stream
                return PIFPAF_OK;
            }
            if (seg[1 + 2 * ns] != 0 || seg[2 + 2 * ns] != 63 || seg[3 + 2 * ns] != 0)
                JPEG_BAD(idx, "bad spectral selection for a sequential scan");
            if (out->w == 0 || out->h == 0) JPEG_BAD(idx, "zero image size");
            if ((int64_t)out->w * out->h > max_pixels) JPEG_BAD(idx, "image over the decoder's pixel capacity");
            std::vector<int> used;
            bool undefined_huff = false;
            for (int i = 0; i < ns; i++) {
                const int cid = seg[1 + 2 * i], tt = seg[2 + 2 * i];
                int ci = -1, hits = 0;
                for (int j = 0; j < nf; j++)
                    if (comps[j].id == cid) { ci = j; hits++; }
                if (hits != 1 || std::find(used.begin(), used.end(), ci) != used.end())
                    JPEG_BAD(idx, "scan component not in the frame");
                used.push_back(ci);
                if ((tt >> 4) > 3 || (tt & 15) > 3) JPEG_BAD(idx, "bad Huffman table selector");
                if (!have_dc[tt >> 4] || !have_ac[tt & 15]) undefined_huff = true;
                if (comps[ci].tq > 3 || !have_q[comps[ci].tq]) JPEG_BAD(idx, "quantisation table missing");
                comps[ci].td = tt >> 4;
                comps[ci].ta = tt & 15;
            }
            // libjpeg-turbo loads its standard tables into an undefined slot (Motion-JPEG frames); libjpeg takes the
            // colour order from the frame and the block order from the scan.  Pillow decodes those streams.
            bool frame_order = true;
            for (int i = 0; i < ns; i++) frame_order = frame_order && used[i] == i;
            if (undefined_huff || !frame_order) {
                out->route = PIFPAF_JPEG_PILLOW;
                return PIFPAF_OK;
            }
            // the entropy-coded bytes: FF00 is a data FF, FF fill bytes belong to the marker after them; RSTn and the
            // codes below SOF0 end a data segment, the first other marker ends the scan
            out->markers.clear();
            int64_t end = -1;
            for (int64_t i = pos; end < 0;) {
                const int64_t a = find_marker(s, i, n, dst, pos, room);
                int64_t j = a;
                while (j < n && s[j] == 0xFF) j++;
                if (j >= n) JPEG_BAD(idx, "no EOI after the scan (truncated stream)");
                for (int64_t k = a; k <= j && k - pos < room; k++) dst[k - pos] = s[k];
                const int c = s[j];
                if (c != 0 && (c < 0xC0 || (c >= 0xD0 && c <= 0xD7))) out->markers.push_back((uint8_t)c);
                else if (c != 0) end = a;
                i = j + 1;
            }
            bool eoi = false;
            for (int64_t i = end; !eoi;) {
                const int64_t a = find_marker(s, i, n);
                if (a + 1 >= n) JPEG_BAD(idx, "no EOI after the scan (truncated stream)");
                eoi = s[a + 1] == 0xD9;
                i = a + 1;
            }
            out->comps.clear();
            for (int ci : used) out->comps.push_back(comps[ci]);
            if (nf == 1) out->comps[0].h = out->comps[0].v = 1;   // not interleaved: one block per MCU
            out->ri = ri;
            out->seg_lo = pos;
            out->seg_hi = end;
            return PIFPAF_OK;
        }
    }
}

}  // namespace

struct pifpaf_jpeg {
    int device;
    int32_t max_images;
    int64_t max_bytes, max_pixels, max_blocks, max_intervals, max_subs, max_chunks;
    std::vector<void*> owned;
    // device
    uint8_t* d_stage;                      // mirror of the pinned staging area
    uint8_t* d_comp;
    int32_t *d_chunk_keep, *d_chunk_rst, *d_comp_len, *d_int_lo, *d_int_hi, *d_int_img, *d_int_sub, *d_int_nsub;
    int32_t *d_int_blocks, *d_seg_lo;
    int32_t *d_sub_int, *d_sub_j, *d_count, *d_acc;
    long long *d_start, *d_exit0, *d_exit1;
    int16_t* d_coef;
    uint8_t* d_plane;
    unsigned long long* d_stats;
    // host
    uint8_t* h_stage;                      // pinned
    int64_t stage_bytes;
    cudaEvent_t staged;
    cudaStream_t last_stream;
    int64_t routes[2];
    int64_t n_subs_last;
};

namespace {

// the last region holds the batch's scan bytes, then (8-byte aligned after them) its interval table
int64_t stage_layout(int64_t max_images, int64_t max_chunks, int64_t max_bytes, int64_t max_intervals, int64_t* off) {
    int64_t o = 0;
    auto take = [&](int64_t bytes) { const int64_t r = o; o = (o + bytes + 255) / 256 * 256; return r; };
    off[0] = take(max_images * sizeof(Img));
    off[1] = take(max_images * 8 * sizeof(Huff));
    off[2] = take(max_images * 4 * 64 * sizeof(int32_t));
    off[3] = take(max_chunks * sizeof(int32_t));
    off[4] = take(max_bytes + 16 + max_intervals * sizeof(int32_t));
    return o;
}

inline int64_t int_table_off(int64_t bytes) { return (bytes + 8 + 7) / 8 * 8; }

// restart interval -> its data segment (segment k follows the k-th marker of the scan; -1: none, the interval decodes
// an empty segment).  libjpeg's read_restart_marker / jpeg_resync_to_restart: interval i > 0 expects
// RST((i - 1) mod 8); the expected marker, or one too far from it, is taken (action 1); a code below SOF0 or one of
// the two RSTs before the expected one is skipped with the data after it (action 2); one of the next two, or the
// scan's end, is left unread (action 3).
void interval_segments(const std::vector<uint8_t>& markers, int n_int, int32_t* out) {
    const int nm = (int)markers.size();
    int cur = 0;
    out[0] = 0;
    for (int i = 1; i < n_int; i++) {
        const int want = (i - 1) & 7;
        out[i] = -1;
        for (;;) {
            const int c = cur < nm ? markers[cur] : 0xD9;
            int action = 1;
            if (c < 0xC0) action = 2;
            else if (c < 0xD0 || c > 0xD7) action = 3;
            else {
                const int dn = (c - 0xD0 - want) & 7;
                action = dn == 1 || dn == 2 ? 3 : dn == 6 || dn == 7 ? 2 : 1;
            }
            if (action == 3) break;
            cur++;
            if (action == 1) { out[i] = cur; break; }
        }
    }
}

inline unsigned grid(long long n, int threads) { return (unsigned)std::max<long long>(1, (n + threads - 1) / threads); }

}  // namespace

extern "C" {

int pifpaf_jpeg_create(pifpaf_jpeg_t** out, int32_t device, int32_t max_images, int64_t max_bytes, int64_t max_pixels,
                       int64_t max_blocks) {
    PIFPAF_CHECK_ARG(out != nullptr, "out is null");
    *out = nullptr;
    PIFPAF_CHECK_ARG(max_images >= 1 && max_bytes >= 1 && max_pixels >= 1 && max_blocks >= 1, "capacities must be positive");
    PIFPAF_CUDA_TRY(cudaSetDevice(device));
    auto* h = new pifpaf_jpeg();
    h->device = device;
    h->max_images = max_images;
    h->max_bytes = max_bytes;
    h->max_pixels = max_pixels;
    h->max_blocks = max_blocks;
    h->max_intervals = max_bytes / 2 + max_images;                      // also bounds the data segments: a marker
                                                                        // takes two bytes
    h->max_subs = max_bytes * 8 / SUBSEQ_BITS + h->max_intervals + max_images;
    h->max_chunks = max_bytes / CHUNK + max_images;
    int64_t off[5];
    h->stage_bytes = stage_layout(max_images, h->max_chunks, max_bytes, h->max_intervals, off);
    int rc = PIFPAF_OK;
    auto alloc = [&](auto** p, size_t n) { if (rc == PIFPAF_OK) rc = pifpaf::dev_alloc(p, n, h->owned); };
    alloc(&h->d_stage, h->stage_bytes);
    alloc(&h->d_comp, max_bytes + 8);
    alloc(&h->d_chunk_keep, h->max_chunks);
    alloc(&h->d_chunk_rst, h->max_chunks);
    alloc(&h->d_comp_len, max_images);
    for (int32_t** p : {&h->d_int_lo, &h->d_int_hi, &h->d_int_img, &h->d_int_sub, &h->d_int_nsub, &h->d_int_blocks,
                        &h->d_seg_lo})
        alloc(p, h->max_intervals);
    for (int32_t** p : {&h->d_sub_int, &h->d_sub_j, &h->d_count, &h->d_acc}) alloc(p, h->max_subs);
    for (long long** p : {&h->d_start, &h->d_exit0, &h->d_exit1}) alloc(p, h->max_subs);
    alloc(&h->d_coef, h->max_blocks * 64);
    alloc(&h->d_plane, h->max_blocks * 64);
    alloc(&h->d_stats, 2);
    if (rc == PIFPAF_OK) {
        const cudaError_t e1 = cudaMallocHost(reinterpret_cast<void**>(&h->h_stage), h->stage_bytes);
        const cudaError_t e2 = e1 == cudaSuccess ? cudaEventCreateWithFlags(&h->staged, cudaEventDisableTiming) : e1;
        if (e1 != cudaSuccess || e2 != cudaSuccess) {
            pifpaf::set_error("pinned staging buffer: %s", cudaGetErrorString(e1 != cudaSuccess ? e1 : e2));
            cudaGetLastError();
            if (e1 == cudaSuccess) cudaFreeHost(h->h_stage);
            h->h_stage = nullptr;
            rc = PIFPAF_E_NOMEM;
        }
    }
    if (rc != PIFPAF_OK) {
        for (void* p : h->owned) cudaFree(p);
        delete h;
        return rc;
    }
    cudaEventRecord(h->staged, 0);
    *out = h;
    return PIFPAF_OK;
}

void pifpaf_jpeg_destroy(pifpaf_jpeg_t* h) {
    if (!h) return;
    cudaSetDevice(h->device);
    cudaDeviceSynchronize();
    for (void* p : h->owned) cudaFree(p);
    if (h->h_stage) cudaFreeHost(h->h_stage);
    cudaEventDestroy(h->staged);
    delete h;
}

int pifpaf_jpeg_decode(pifpaf_jpeg_t* h, int32_t n, const uint8_t* const* data, const int64_t* sizes,
                       uint8_t* out_dev, int64_t out_bytes, int32_t max_rounds,
                       int32_t* routes, int32_t* hw, int64_t* out_offsets, void* stream_v) {
    PIFPAF_CHECK_ARG(h != nullptr && data != nullptr && sizes != nullptr && routes && hw && out_offsets, "null argument");
    PIFPAF_CHECK_ARG(n >= 0 && n <= h->max_images, "more images than the handle's max_images");
    PIFPAF_CHECK_ARG(out_dev != nullptr || n == 0, "output buffer is null");
    PIFPAF_CHECK_ARG(max_rounds >= -1 && max_rounds <= 1024, "max_rounds must be -1 (default) or 0..1024");
    if (max_rounds < 0) max_rounds = DEFAULT_ROUNDS;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_v);
    PIFPAF_CUDA_TRY(cudaSetDevice(h->device));
    PIFPAF_CUDA_TRY(cudaEventSynchronize(h->staged));      // the previous batch's staging copy has been read
    int64_t off[5];
    stage_layout(h->max_images, h->max_chunks, h->max_bytes, h->max_intervals, off);
    Img* imgs = reinterpret_cast<Img*>(h->h_stage + off[0]);
    Huff* tabs = reinterpret_cast<Huff*>(h->h_stage + off[1]);
    int32_t* quant = reinterpret_cast<int32_t*>(h->h_stage + off[2]);
    int32_t* chunk_img = reinterpret_cast<int32_t*>(h->h_stage + off[3]);
    uint8_t* raw = h->h_stage + off[4];
    // pass 1: parse and validate everything; nothing is launched or copied unless every stream is accepted
    int n_gpu = 0;
    int64_t bytes = 0, chunks = 0, blocks = 0, px = 0, out = 0, intervals = 0, subs = 0, segs = 0;
    std::vector<Parsed> ps(n);
    for (int i = 0; i < n; i++) {
        PIFPAF_CHECK_ARG(data[i] != nullptr && sizes[i] >= 0, "null stream");
        Parsed& p = ps[i];
        PIFPAF_TRY(parse_jpeg(i, data[i], sizes[i], h->max_pixels, tabs + 8 * n_gpu, quant + 4 * 64 * n_gpu, raw + bytes,
                              h->max_bytes + 16 - bytes, &p));
        routes[i] = p.route;
        hw[2 * i] = p.route == PIFPAF_JPEG_GPU ? p.h : 0;
        hw[2 * i + 1] = p.route == PIFPAF_JPEG_GPU ? p.w : 0;
        out_offsets[i] = -1;
        if (p.route != PIFPAF_JPEG_GPU) continue;
        Img& im = imgs[n_gpu];
        std::memset(&im, 0, sizeof(Img));
        im.w = p.w;
        im.h = p.h;
        im.ncomp = (int)p.comps.size();
        im.hmax = im.vmax = 1;
        for (const Comp& c : p.comps) { im.hmax = std::max(im.hmax, c.h); im.vmax = std::max(im.vmax, c.v); }
        im.mx = (p.w + 8 * im.hmax - 1) / (8 * im.hmax);
        im.my = (p.h + 8 * im.vmax - 1) / (8 * im.vmax);
        const int64_t n_mcu = (int64_t)im.mx * im.my;
        im.ri = p.ri ? p.ri : (int32_t)n_mcu;
        im.n_int = (int32_t)((n_mcu + im.ri - 1) / im.ri);
        int b = 0;
        for (int c = 0; c < im.ncomp; c++) {
            const Comp& cc = p.comps[c];
            im.comp_h[c] = cc.h;
            im.comp_v[c] = cc.v;
            im.comp_first[c] = b;
            for (int v = 0; v < cc.v; v++)
                for (int hh = 0; hh < cc.h; hh++, b++) { im.blk_comp[b] = c; im.blk_v[b] = v; im.blk_h[b] = hh; }
            im.plane_w[c] = im.mx * cc.h * 8;
            im.plane_h[c] = im.my * cc.v * 8;
            im.huff[c][0] = 8 * n_gpu + cc.td;
            im.huff[c][1] = 8 * n_gpu + 4 + cc.ta;
            im.quant[c] = 4 * n_gpu + cc.tq;
        }
        im.bpm = b;
        // planes: component c after the planes of the components before it
        int64_t po = blocks * 64;
        for (int c = 0; c < im.ncomp; c++) {
            im.plane_off[c] = po;
            po += (int64_t)im.plane_w[c] * im.plane_h[c];
        }
        im.seg_len = (int32_t)(p.seg_hi - p.seg_lo);
        if (p.seg_hi - p.seg_lo > (int64_t)INT32_MAX / 8) JPEG_BAD(i, "scan over 256 MB");
        im.seg_off = bytes;
        im.n_chunks = (im.seg_len + CHUNK - 1) / CHUNK;
        im.chunk_base = (int32_t)chunks;
        im.int_base = (int32_t)intervals;
        im.seg_base = (int32_t)segs;
        im.n_seg = (int32_t)p.markers.size() + 1;
        im.sub_base = (int32_t)subs;
        im.sub_cap = (int32_t)(((int64_t)im.seg_len * 8 + SUBSEQ_BITS - 1) / SUBSEQ_BITS + im.n_int);
        im.blk_base = blocks;
        im.px_base = px;
        im.out_off = out;
        bytes += im.seg_len;
        chunks += im.n_chunks;
        intervals += im.n_int;
        segs += im.n_seg;
        subs += im.sub_cap;
        blocks += n_mcu * im.bpm;
        px += (int64_t)p.w * p.h;
        out += (int64_t)p.w * p.h * 3;
        if (bytes > h->max_bytes) JPEG_BAD(i, "the batch's scan data exceeds the handle's max_bytes");
        if (blocks > h->max_blocks) JPEG_BAD(i, "the batch's 8x8 blocks exceed the handle's max_blocks");
        if (intervals > h->max_intervals || segs > h->max_intervals || subs > h->max_subs || chunks > h->max_chunks)
            JPEG_BAD(i, "the batch's restart intervals exceed the handle's capacity");
        if (out > out_bytes) JPEG_BAD(i, "the output buffer is too small for the batch");
        out_offsets[i] = im.out_off;
        n_gpu++;
    }
    h->routes[0] = n_gpu;
    h->routes[1] = n - n_gpu;
    h->n_subs_last = subs;
    h->last_stream = st;
    PIFPAF_CUDA_TRY(cudaMemsetAsync(h->d_stats, 0, 2 * sizeof(unsigned long long), st));
    if (n_gpu == 0) return PIFPAF_OK;
    // pass 2: stage the chunk table and the interval table (the scan bytes were staged by the walk), one copy
    int32_t* int_seg = reinterpret_cast<int32_t*>(raw + int_table_off(bytes));
    for (int i = 0, g = 0; i < n; i++) {
        if (ps[i].route != PIFPAF_JPEG_GPU) continue;
        const Img& im = imgs[g];
        for (int c = 0; c < im.n_chunks; c++) chunk_img[im.chunk_base + c] = g;
        interval_segments(ps[i].markers, im.n_int, int_seg + im.int_base);
        g++;
    }
    PIFPAF_CUDA_TRY(cudaMemcpyAsync(h->d_stage, h->h_stage, off[4] + int_table_off(bytes) + intervals * sizeof(int32_t),
                                    cudaMemcpyHostToDevice, st));
    PIFPAF_CUDA_TRY(cudaEventRecord(h->staged, st));

    Dev d;
    d.img = reinterpret_cast<const Img*>(h->d_stage + off[0]);
    d.huff = reinterpret_cast<const Huff*>(h->d_stage + off[1]);
    d.quant = reinterpret_cast<const int32_t*>(h->d_stage + off[2]);
    d.chunk_img = reinterpret_cast<const int32_t*>(h->d_stage + off[3]);
    d.raw = h->d_stage + off[4];
    d.int_seg = reinterpret_cast<const int32_t*>(d.raw + int_table_off(bytes));
    d.seg_lo = h->d_seg_lo;
    d.int_blocks = h->d_int_blocks;
    d.comp = h->d_comp;
    d.chunk_keep = h->d_chunk_keep; d.chunk_rst = h->d_chunk_rst; d.comp_len = h->d_comp_len;
    d.int_lo = h->d_int_lo; d.int_hi = h->d_int_hi; d.int_img = h->d_int_img; d.int_sub = h->d_int_sub;
    d.int_nsub = h->d_int_nsub;
    d.sub_int = h->d_sub_int; d.sub_j = h->d_sub_j; d.start = h->d_start; d.exit0 = h->d_exit0; d.exit1 = h->d_exit1;
    d.count = h->d_count; d.acc = h->d_acc;
    d.coef = h->d_coef; d.plane = h->d_plane; d.out = out_dev; d.stats = h->d_stats;

    k_jpeg_unstuff_count<<<grid(chunks, 256), 256, 0, st>>>(d, (int)chunks);
    PIFPAF_LAUNCH_CHECK();
    k_jpeg_unstuff_scan<<<n_gpu, 1024, 0, st>>>(d);
    PIFPAF_LAUNCH_CHECK();
    k_jpeg_unstuff_write<<<grid(chunks, 256), 256, 0, st>>>(d, (int)chunks);
    PIFPAF_LAUNCH_CHECK();
    k_jpeg_subseq_setup<<<n_gpu, 1024, 0, st>>>(d);
    PIFPAF_LAUNCH_CHECK();
    for (int r = 0; r < max_rounds; r++) {
        k_jpeg_sync<<<grid(subs, 128), 128, 0, st>>>(d, (int)subs, r);
        PIFPAF_LAUNCH_CHECK();
    }
    k_jpeg_settle<<<grid(intervals * 32, 128), 128, 0, st>>>(d, (int)intervals, max_rounds > 0 ? (max_rounds - 1) & 1 : 0);
    PIFPAF_LAUNCH_CHECK();
    PIFPAF_CUDA_TRY(cudaMemsetAsync(h->d_coef, 0, blocks * 64 * sizeof(int16_t), st));
    k_jpeg_write<<<grid(subs, 128), 128, 0, st>>>(d, (int)subs);
    PIFPAF_LAUNCH_CHECK();
    k_jpeg_dc<<<3 * n_gpu, 1024, 0, st>>>(d);
    PIFPAF_LAUNCH_CHECK();
    k_jpeg_idct<<<grid(blocks, 128), 128, 0, st>>>(d, n_gpu, blocks);
    PIFPAF_LAUNCH_CHECK();
    k_jpeg_color<<<grid(px, 256), 256, 0, st>>>(d, n_gpu, px);
    PIFPAF_LAUNCH_CHECK();
    return PIFPAF_OK;
}

int pifpaf_jpeg_last_stats(pifpaf_jpeg_t* h, int64_t* stats, int32_t n_stats) {
    PIFPAF_CHECK_ARG(h != nullptr && stats != nullptr && n_stats >= 0, "null argument");
    unsigned long long dev[2] = {0, 0};
    PIFPAF_CUDA_TRY(cudaSetDevice(h->device));
    PIFPAF_CUDA_TRY(cudaStreamSynchronize(h->last_stream));
    PIFPAF_CUDA_TRY(cudaMemcpy(dev, h->d_stats, sizeof(dev), cudaMemcpyDeviceToHost));
    const int64_t all[5] = {h->routes[0], h->routes[1], h->n_subs_last, (int64_t)dev[0], (int64_t)dev[1]};
    for (int i = 0; i < n_stats; i++) stats[i] = i < 5 ? all[i] : 0;
    return PIFPAF_OK;
}

}  // extern "C"
