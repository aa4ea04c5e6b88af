// libpifpaf_b200 -- backbone + heads forward for sm_90a (H100).
//
// Replaces the cuDNN/ATen kernels behind the reference's torch.nn modules
// (paths relative to the reference's src/openpifpaf/):
//   Shell.forward                 network/nets.py:35-48
//   ShuffleNetV2K/InvertedResidualK   network/basenetworks.py:186-355
//   CompositeField4 (eval)        network/heads.py:330-378
//
// Activations are NHWC bf16 ("rows" = pixels, "columns" = channels).  Every 1x1
// convolution (97 % of the MACs of shufflenetv2k16) is one GEMM
//   out[M = B*H*W, N] = act[M, K] * W[N, K]^T,  f32 accumulate
// executed by k_gemm_wg: a persistent, warp-specialised wgmma kernel -- one
// producer lane streams TMA tiles (128B swizzle) through a shared-memory ring,
// two consumer warpgroups each own 64 rows of the 128-row tile, accumulate it in
// registers with wgmma.mma_async and run the epilogue (bias + ReLU, bf16) that
// also fuses torch.cat + channel_shuffle(2) (interleaving with the pass-through
// half) or the CompositeField4 eval epilogue (sigmoid, index-field add,
// softplus, f32 [B,F,comp,h,w] layout).
// Depthwise 5x5 and the 3-channel input conv are bandwidth-bound direct kernels.
#include <cuda.h>
#include <cuda_bf16.h>

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <utility>
#include <vector>

#include "common.cuh"

namespace {

// ------------------------------------------------------------------ PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) {}
}
__device__ __forceinline__ void fence_barrier_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* map, uint64_t* bar,
                                            int c0, int c1, int c2, int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)),
          "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}
// shared -> global tensor store (bulk async-group completion, tracked per issuing thread)
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, const void* smem_src, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
                 ::"l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
                 : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// all but the newest PENDING bulk groups of this thread have finished reading shared memory
template <int PENDING>
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(PENDING) : "memory"); }
// all bulk groups of this thread have completed (their global writes are done)
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
// orders generic-proxy shared-memory writes before the async proxy (TMA, wgmma) reads them
__device__ __forceinline__ void fence_proxy_async_shared() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// ---- warpgroup MMA (wgmma): D[registers] (+)= A[smem] * B[smem]^T, bf16 inputs, f32 accumulate, issued by the four
// warps of a warpgroup together.  m64nNk16: thread t of the warpgroup holds, for every group of 8 columns,
// d[4j], d[4j+1] = row 16 * (warp % 4) + lane / 4, columns 8j + 2 * (lane % 4) + {0, 1}; d[4j+2], d[4j+3] = 8 rows below.
// register budget of a warp-specialised kernel: a warpgroup lowers or raises its per-thread limit (multiple of 8)
template <int REGS>
__device__ __forceinline__ void reg_dealloc() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(REGS)); }
template <int REGS>
__device__ __forceinline__ void reg_alloc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(REGS)); }
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int PENDING>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(PENDING) : "memory"); }
// keeps every use of the accumulator registers on its side of the asynchronous MMAs
template <int N>
__device__ __forceinline__ void fence_acc(float (&d)[N]) {
#pragma unroll
    for (int i = 0; i < N; i++) asm volatile("" : "+f"(d[i])::"memory");
}
__device__ __forceinline__ void wgmma_n16(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(adesc), "l"(bdesc), "r"(accumulate)
        : "memory");
}
__device__ __forceinline__ void wgmma_n32(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(adesc), "l"(bdesc), "r"(accumulate)
        : "memory");
}
__device__ __forceinline__ void wgmma_n48(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %26, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n48k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23}, %24, %25, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
        : "l"(adesc), "l"(bdesc), "r"(accumulate)
        : "memory");
}
__device__ __forceinline__ void wgmma_n64(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(adesc), "l"(bdesc), "r"(accumulate)
        : "memory");
}
// one 64-column group (or the narrower last group: N = 16, 32, 48) of a k16 step.  N is a compile-time constant:
// a wgmma behind a runtime branch makes ptxas fence every one of them (warpgroup.arrive, C7519)
template <int N>
__device__ __forceinline__ void wgmma_group(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    static_assert(N == 16 || N == 32 || N == 48 || N == 64, "wgmma group width");
    if constexpr (N == 64) wgmma_n64(d, adesc, bdesc, accumulate);
    else if constexpr (N == 48) wgmma_n48(d, adesc, bdesc, accumulate);
    else if constexpr (N == 32) wgmma_n32(d, adesc, bdesc, accumulate);
    else wgmma_n16(d, adesc, bdesc, accumulate);
}

// Programmatic dependent launch (PDL): a kernel launched with cudaLaunchAttributeProgrammaticStreamSerialization may
// start while its predecessor in the stream is still draining; everything up to pdl_wait() (barrier init,
// descriptor prefetch, staging of constant weights / biases) overlaps the predecessor's tail.
// pdl_wait() returns once the predecessor has completed and its writes are visible -- it must precede every access
// to activations (reads AND writes: the predecessor may still be reading what this kernel overwrites).  Both are
// no-ops in a kernel launched the ordinary way.
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// ------------------------------------------------------------------ descriptors
constexpr int BM = 128;          // tile rows: two consumer warpgroups x 64 (wgmma M)
constexpr int BK = 64;           // one 128-byte swizzle atom of bf16 per smem row
constexpr int MMA_K = 16;
constexpr int WG_ROWS = 64;      // rows per consumer warpgroup
constexpr int NGROUP = 64;       // columns per wgmma instruction (the last group of a tile may be 16, 32 or 48)
constexpr int CONSUMER_WARPS = 8;
constexpr int GEMM_THREADS = 128 + 32 * CONSUMER_WARPS;   // warpgroup 0: TMA producer (one lane); warpgroups 1, 2: MMA + epilogue
constexpr int CHUNK = 16;        // epilogue column chunk (one lane: one row x 16 columns)
constexpr int STG_LD = 33;       // row pitch (words) of a warp's 16 x 32 accumulator staging tile: reads (one row per lane)
                                 // are conflict-free, the fragment-order writes see 2-way conflicts
constexpr int STG_BYTES = CONSUMER_WARPS * 16 * STG_LD * 4;

// K-major, SWIZZLE_128B shared-memory matrix descriptor of wgmma:
// start>>4 | LBO(ignored for swizzled K-major)=1 @16 | SBO = 1024 B (8 rows x 128 B) >>4 @32 | layout 128B swizzle (1) @62
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= static_cast<uint64_t>((smem_addr >> 4) & 0x3fffu);
    d |= static_cast<uint64_t>(1u) << 16;
    d |= static_cast<uint64_t>(1024u >> 4) << 32;
    d |= static_cast<uint64_t>(1u) << 62;
    return d;
}

// ------------------------------------------------------------------ GEMM arguments
enum { MODE_PLAIN = 0, MODE_SHUFFLE = 1, MODE_HEADS = 2, MODE_SCATTER = 3 };

// MODE_SCATTER: destination of one chunk of 16 GEMM columns (32 bytes per row, one 256-bit store per lane): base
// already points at the chunk's first column inside its tensor (a multiple of 16 channels)
// store: the same destination for the TMA-store epilogue, (store map index << 16) | first column inside that map
struct DestGroup { __nv_bfloat16* base; int ld; int store; };
static_assert(sizeof(DestGroup) == 16, "DestGroup is copied to shared memory as 16-byte entries");

// TMA-store epilogue (MODE_PLAIN without residual, MODE_SCATTER): output tensor maps, rows bounded at the forward's
// batch * h * w.  Plain: map 0 = the output window.  Scatter: one map per destination tensor.
constexpr int MAX_STORE_MAPS = 8;
struct StoreMaps { CUtensorMap m[MAX_STORE_MAPS]; };
constexpr int OUT_BOX_COLS = 16, OUT_BOX_ROWS = 16;      // one box: a warp's 16 rows x 16 columns, 32-byte swizzle
constexpr int OUT_BOX_BYTES = OUT_BOX_ROWS * OUT_BOX_COLS * 2;
constexpr int OUT_CHUNK_BYTES = 2 * OUT_BOX_BYTES;       // 32 columns: half of a wgmma column group
constexpr int OUT_WARP_BYTES = 2 * OUT_CHUNK_BYTES;      // double buffered
static_assert(CONSUMER_WARPS * OUT_WARP_BYTES <= STG_BYTES, "the output chunks live in the f32 staging region");

// per GEMM output column (heads mode): plane = field * n_comp + comp; sub = (dy << 8) | dx is the PixelShuffle
// position of this conv channel inside the up x up block of its cell (heads.py:333-343), 0 without upsampling
struct HeadCol { int head; int plane; int op; int sub; };

struct GemmArgs {
    int M, N, K;                 // rows, real output channels, k extent (columns of the A view)
    int a_col0;                  // first column of the A view inside its tensor (TMA coordinate; multiple of 8)
    int block_n, n_blocks, m_blocks, num_k_blocks, stages;
    int mode, relu;
    const float* bias;           // [n_blocks * block_n], zero padded
    // plain / shuffle
    __nv_bfloat16* out; int ldo; int out_col_off;
    const __nv_bfloat16* src0; int ld0; int src0_col_off; int half; int gap;
    int src_tma;                 // pass-through tile arrives by TMA in shared memory (else read from global)
    int b_resident;              // all K blocks of this CTA's weight tile stay in shared memory (loaded once)
    int tma_store;               // epilogue through shared memory + TMA stores (StoreMaps), else per-lane global stores
    // scatter: chunks of 16 columns go to different tensors (the 'bins' layout: every channel is written once,
    // into the buffer of the block that consumes it)
    const DestGroup* dest;       // [n_blocks * block_n / 16]
    // heads
    const HeadCol* head_cols;    // [n_blocks * block_n]
    float* head_base[4]; int head_planes[4];
    int hw, w;                   // pixels per image, field width (of the conv output)
    int up, up_low, out_h, out_w;   // PixelShuffle factor, low crop, head output size (== h, w when up == 1)
    // implicit-GEMM convolution (conv_k > 0): one M tile = a PH x PW patch of output pixels of one image;
    // K blocks run over taps x 64-channel blocks; A comes from a 4-D tensor map {C, W, H, B}; tap t reads input
    // pixel (x * stride - pad + (t % k) * dil, y * stride - pad + (t / k) * dil)
    int conv_k, conv_stride, conv_pad, conv_dil, conv_cblocks;
    int Hi, Wi, Ho, Wo, tiles_x, tiles_y;
    // residual add before the ReLU (torchvision BasicBlock / Bottleneck): res[m][res_col_off + n]
    const __nv_bfloat16* res; int ld_res; int res_col_off;
    // debug (SIMT) operand views
    const __nv_bfloat16* a; int lda; const __nv_bfloat16* wgt; int ldw;
};

constexpr int PH = 8, PW = 16;     // conv output patch per M tile (PH * PW == BM)

// tile row -> output row index m, or -1 if outside the tensor
__device__ __forceinline__ int tile_row_to_m(const GemmArgs& g, int m_blk, int row) {
    if (g.conv_k == 0) {
        const int m = m_blk * BM + row;
        return m < g.M ? m : -1;
    }
    const int per_img = g.tiles_x * g.tiles_y;
    const int b = m_blk / per_img, t = m_blk - b * per_img;
    const int oy = (t / g.tiles_x) * PH + row / PW, ox = (t % g.tiles_x) * PW + row % PW;
    if (oy >= g.Ho || ox >= g.Wo) return -1;
    return (b * g.Ho + oy) * g.Wo + ox;
}

__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
    __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float softplus_f(float x) {   // torch softplus beta=1 threshold=20 (heads.py:378)
    return x > 20.0f ? x : log1pf(expf(x));
}
__device__ __forceinline__ float sigmoid_f(float x) { return 1.0f / (1.0f + expf(-x)); }

// activation code of the conv entry points (include/pifpaf_b200.h): 0 none, 1 ReLU, 2 ReLU6 (MobileNetV2,
// torchvision's ReLU6 = hardtanh(x, 0, 6); exact in f32 and after rounding to bf16, 6 is a bf16 value)
constexpr int ACT_NONE = 0, ACT_RELU = 1, ACT_RELU6 = 2;
__device__ __forceinline__ float act_f(float x, int act) {
    if (act) {
        x = fmaxf(x, 0.f);
        if (act == ACT_RELU6) x = fminf(x, 6.f);
    }
    return x;
}

// 32 bytes (one sector) as two 128-bit global stores: p must be 32-byte aligned
__device__ __forceinline__ void st_global_256(void* p, uint32_t a, uint32_t b, uint32_t c, uint32_t d,
                                              uint32_t e, uint32_t f, uint32_t g, uint32_t h) {
    uint4* q = reinterpret_cast<uint4*>(p);
    q[0] = make_uint4(a, b, c, d);
    q[1] = make_uint4(e, f, g, h);
}

// store `cnt` (<= 16) consecutive 32-bit words from registers to p (4-byte aligned, LEAD words before the
// first 16-byte boundary): scalar lead-in, 16-byte vectors, scalar tail.  Fully unrolled (no local memory).
template <int LEAD>
__device__ __forceinline__ void store_words(uint32_t* p, const uint32_t (&w)[CHUNK], int cnt) {
#pragma unroll
    for (int i = 0; i < LEAD; i++)
        if (i < cnt) p[i] = w[i];
#pragma unroll
    for (int i = LEAD; i + 4 <= CHUNK; i += 4) {
        if (i + 4 <= cnt) {
            *reinterpret_cast<uint4*>(p + i) = make_uint4(w[i], w[i + 1], w[i + 2], w[i + 3]);
        } else {
#pragma unroll
            for (int j = 0; j < 4; j++)
                if (i + j < cnt) p[i + j] = w[i + j];
        }
    }
#pragma unroll
    for (int i = LEAD + (CHUNK - LEAD) / 4 * 4; i < CHUNK; i++)
        if (i < cnt) p[i] = w[i];
}

// Epilogue for one warp: 32 rows (lane == row) x CHUNK columns starting at GEMM column n0.
// acc[] holds this lane's CHUNK accumulators.  Every lane writes its own row with 16-byte vector stores
// (full 32-byte sectors), no shared-memory staging.
// bias: pointer to this chunk's CHUNK biases (shared memory in the tensor-core kernel, global in the debug
// kernel).  src_row: this lane's row of the pass-through tile at the chunk's first column (shared memory, filled
// by TMA) or nullptr to read it from global memory.
// dest: the MODE_SCATTER destination table (shared memory in the tensor-core kernel: a global load per chunk put
// stalls every epilogue warp; global in the debug kernel)
__device__ __forceinline__ void epilogue_chunk(const GemmArgs& g, int m, int n0, const float* acc,
                                               const float* bias, const __nv_bfloat16* src_row,
                                               const DestGroup* dest) {
    float bv[CHUNK];
    {
        const float4* bp = reinterpret_cast<const float4*>(bias);
#pragma unroll
        for (int j = 0; j < CHUNK / 4; j++) {
            const float4 b4 = bp[j];
            bv[4 * j] = b4.x; bv[4 * j + 1] = b4.y; bv[4 * j + 2] = b4.z; bv[4 * j + 3] = b4.w;
        }
    }
    if (m < 0) return;
    if (g.mode == MODE_HEADS) {
        const int b = m / g.hw, pix = m - b * g.hw;
        const int y = pix / g.w, x = pix - y * g.w;
        const int out_hw = g.out_h * g.out_w;
#pragma unroll
        for (int j = 0; j < CHUNK; j++) {
            const int n = n0 + j;
            if (n >= g.N) break;
            const HeadCol hc = g.head_cols[n];
            // PixelShuffle(up) + crop [low, size - high) (heads.py:333-343): conv channel c*up*up + dy*up + dx of
            // cell (y, x) is output channel c at (y*up + dy - low, x*up + dx - low)
            const int oy = y * g.up + (hc.sub >> 8) - g.up_low, ox = x * g.up + (hc.sub & 255) - g.up_low;
            if (oy < 0 || oy >= g.out_h || ox < 0 || ox >= g.out_w) continue;
            float v = acc[j] + bv[j];
            if (hc.op == 1) v = sigmoid_f(v);
            else if (hc.op == 2) v += (float)ox;
            else if (hc.op == 3) v += (float)oy;
            else if (hc.op == 4) v = softplus_f(v);
            g.head_base[hc.head][((size_t)b * g.head_planes[hc.head] + hc.plane) * out_hw + oy * g.out_w + ox] = v;
        }
        return;
    }
    if (g.mode == MODE_SCATTER) {
        uint32_t w[CHUNK / 2];
#pragma unroll
        for (int j = 0; j < CHUNK; j += 2) {
            float a0 = acc[j] + bv[j], a1 = acc[j + 1] + bv[j + 1];
            if (g.relu) { a0 = fmaxf(a0, 0.f); a1 = fmaxf(a1, 0.f); }
            w[j >> 1] = pack_bf16(a0, a1);
        }
        if (n0 < g.N) {
            const DestGroup d = dest[n0 >> 4];
            st_global_256(d.base + (size_t)m * d.ld, w[0], w[1], w[2], w[3], w[4], w[5], w[6], w[7]);
        }
        return;
    }
    if (g.mode == MODE_PLAIN) {
        uint32_t w[CHUNK / 2];
        float rv[CHUNK];
        if (g.res != nullptr) {
            const uint4* rp = reinterpret_cast<const uint4*>(g.res + (size_t)m * g.ld_res + g.res_col_off + n0);
            const uint4 r0 = __ldg(rp), r1 = __ldg(rp + 1);
            const uint32_t rw[8] = {r0.x, r0.y, r0.z, r0.w, r1.x, r1.y, r1.z, r1.w};
#pragma unroll
            for (int j = 0; j < 8; j++) {
                rv[2 * j] = __uint_as_float(rw[j] << 16);
                rv[2 * j + 1] = __uint_as_float(rw[j] & 0xffff0000u);
            }
        } else {
#pragma unroll
            for (int j = 0; j < CHUNK; j++) rv[j] = 0.f;
        }
#pragma unroll
        for (int j = 0; j < CHUNK; j += 2) {
            float a0 = acc[j] + bv[j] + rv[j], a1 = acc[j + 1] + bv[j + 1] + rv[j + 1];
            if (g.relu) { a0 = fmaxf(a0, 0.f); a1 = fmaxf(a1, 0.f); }
            if (g.relu == ACT_RELU6) { a0 = fminf(a0, 6.f); a1 = fminf(a1, 6.f); }
            w[j >> 1] = pack_bf16(a0, a1);
        }
        // 16 bf16 = 32 bytes, 32-byte aligned (ldo % 16 == 0, out_col_off % 16 == 0, n0 % 16 == 0)
        uint4* dst = reinterpret_cast<uint4*>(g.out + (size_t)m * g.ldo + g.out_col_off + n0);
        const int n_pad8 = (g.N + 7) & ~7;
        if (n0 + 8 < n_pad8) {
            st_global_256(dst, w[0], w[1], w[2], w[3], w[4], w[5], w[6], w[7]);
        } else if (n0 < n_pad8) {
            dst[0] = make_uint4(w[0], w[1], w[2], w[3]);
        }
        return;
    }
    // MODE_SHUFFLE: word n = { src0[m][n] (logical channel 2n), conv[m][n] (logical 2n+1) }
    const uint4* sp = src_row != nullptr
        ? reinterpret_cast<const uint4*>(src_row)
        : reinterpret_cast<const uint4*>(g.src0 + (size_t)m * g.ld0 + g.src0_col_off + n0);
    const uint4 s0 = sp[0], s1 = sp[1];
    const uint32_t sw[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
    uint32_t w[CHUNK];
#pragma unroll
    for (int j = 0; j < CHUNK; j++) {
        float a = acc[j] + bv[j];
        if (g.relu) a = fmaxf(a, 0.f);
        const uint32_t src_bits = (j & 1) ? (sw[j >> 1] >> 16) : (sw[j >> 1] & 0xffffu);
        const __nv_bfloat16 hb = __float2bfloat16_rn(a);
        w[j] = src_bits | (static_cast<uint32_t>(__bfloat16_as_ushort(hb)) << 16);
    }
    // logical channel 2n, 2n+1 == physical word n (gap-free layout): 64 bytes per lane, 64-byte aligned
    uint32_t* row = reinterpret_cast<uint32_t*>(g.out) + (size_t)m * (g.ldo >> 1) + (g.out_col_off >> 1) + n0;
    const int cnt = min(CHUNK, g.N - n0);
    if (cnt == CHUNK) {
        st_global_256(row, w[0], w[1], w[2], w[3], w[4], w[5], w[6], w[7]);
        st_global_256(row + 8, w[8], w[9], w[10], w[11], w[12], w[13], w[14], w[15]);
    } else {
        store_words<0>(row, w, cnt);
    }
}

// ------------------------------------------------------------------ consumer side shared by the wgmma kernels
// D (+)= A-tile rows [64 * wg, +64) x B-tile^T over one 64-wide K block: 4 k16 steps x NG column groups, the last
// LASTW (16, 32, 48 or 64) columns wide -- the tile is (NG - 1) * 64 + LASTW columns
template <int NG, int LASTW>
__device__ __forceinline__ void mma_k_block(float (&acc)[NG][32], uint32_t sa, uint32_t sb, bool first) {
#pragma unroll
    for (int k = 0; k < BK / MMA_K; k++) {
        const uint64_t adesc = make_smem_desc(sa + k * MMA_K * 2);
        const uint32_t accumulate = (first && k == 0) ? 0u : 1u;
#pragma unroll
        for (int gi = 0; gi < NG - 1; gi++)
            wgmma_group<NGROUP>(acc[gi], adesc, make_smem_desc(sb + gi * NGROUP * BK * 2 + k * MMA_K * 2), accumulate);
        wgmma_group<LASTW>(acc[NG - 1], adesc, make_smem_desc(sb + (NG - 1) * NGROUP * BK * 2 + k * MMA_K * 2),
                           accumulate);
    }
}

// Epilogue of one consumer warp: its 16 rows x block_n accumulators go through a 16 x 32 shared-memory tile so that a
// lane holds one row x 16 consecutive columns (what epilogue_chunk stores as whole 32-byte sectors): lanes 0-15 take
// the first 16 columns of a 32-column piece, lanes 16-31 the second.
// row0: first tile row of this warp; src_tile: pass-through tile [BM][block_n] in shared memory or nullptr
template <int NG>
__device__ __forceinline__ void warp_epilogue(const GemmArgs& g, float (&acc)[NG][32], float* stg, int m_blk, int n_blk,
                                              int row0, const float* bias_s, const __nv_bfloat16* src_tile,
                                              const DestGroup* dest_s) {
    const int lane = threadIdx.x & 31;
    const int r = lane >> 2, q = lane & 3;
    const int er = lane & 15, ec = lane >> 4;
    const int m = tile_row_to_m(g, m_blk, row0 + er);
#pragma unroll
    for (int gi = 0; gi < NG; gi++) {
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int p = gi * NGROUP + h * 32;
            if (p >= g.block_n) continue;
#pragma unroll
            for (int t = 0; t < 4; t++) {
                const int tt = h * 4 + t;
                stg[r * STG_LD + 8 * t + 2 * q] = acc[gi][4 * tt];
                stg[r * STG_LD + 8 * t + 2 * q + 1] = acc[gi][4 * tt + 1];
                stg[(r + 8) * STG_LD + 8 * t + 2 * q] = acc[gi][4 * tt + 2];
                stg[(r + 8) * STG_LD + 8 * t + 2 * q + 1] = acc[gi][4 * tt + 3];
            }
            __syncwarp();
            const int c = p + ec * CHUNK;
            const int n0 = n_blk * g.block_n + c;
            if (c < g.block_n && n0 < ((g.N + 7) & ~7)) {
                float accf[CHUNK];
#pragma unroll
                for (int j = 0; j < CHUNK; j++) accf[j] = stg[er * STG_LD + ec * CHUNK + j];
                epilogue_chunk(g, m, n0, accf, bias_s + n0,
                               src_tile != nullptr ? src_tile + (size_t)(row0 + er) * g.block_n + c : nullptr, dest_s);
            }
            __syncwarp();
        }
    }
}

// TMA-store epilogue of one consumer warp (MODE_PLAIN without residual, MODE_SCATTER): its 16 rows x BN accumulators
// go, with bias and ReLU, as bf16 straight from the wgmma fragments into 16 x 16 boxes in shared memory (32-byte
// swizzle: a row's two 16-byte halves swap on rows 4-7 of every 8, which makes the fragment-order writes
// conflict-free), and one lane stores every box with a TMA tensor store.  The warp does not wait for the stores: it
// goes on to the next tile's MMAs, and reclaims a 32-column chunk buffer (two boxes) only when the bulk group that
// read it two chunks ago has finished reading.  The tensor maps clip rows at M and, in plain mode, columns at the
// window's pad8(N), so rows past the batch and columns past the window are never written.
// obuf: this warp's two chunk buffers; ob: which of them is next (carried across tiles)
template <int NG, int LASTW>
__device__ __forceinline__ void warp_epilogue_tma(const GemmArgs& g, const StoreMaps& maps, float (&acc)[NG][32],
                                                  unsigned char* obuf, int& ob, int m_blk, int n_blk, int row0,
                                                  const float* bias_s, const DestGroup* dest_s) {
    constexpr int BN = (NG - 1) * NGROUP + LASTW;
    const int lane = threadIdx.x & 31;
    const int r = lane >> 2, q = lane & 3;
    const int sw = (r >> 2) & 1;                       // rows r and r + 8 share it
    const int m0 = m_blk * BM + row0;
    const float* bias_t = bias_s + n_blk * BN;
    const int n_lim = g.mode == MODE_SCATTER ? g.N : ((g.N + 7) & ~7);
#pragma unroll
    for (int gi = 0; gi < NG; gi++) {
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int p = gi * NGROUP + h * 32;        // first tile column of this chunk
            if (p >= BN) continue;
            const int boxes = (BN - p) >= 32 ? 2 : 1;  // compile-time after unrolling
            unsigned char* buf = obuf + ob * OUT_CHUNK_BYTES;
            if (lane == 0) bulk_wait_read<1>();
            __syncwarp();
#pragma unroll
            for (int t = 0; t < 4; t++) {
                if (t >= 2 * boxes) continue;
                const int j = h * 4 + t;               // 8-column fragment group inside the wgmma group
                const float2 b = *reinterpret_cast<const float2*>(bias_t + p + 8 * t + 2 * q);
                float v0 = acc[gi][4 * j] + b.x, v1 = acc[gi][4 * j + 1] + b.y;
                float v2 = acc[gi][4 * j + 2] + b.x, v3 = acc[gi][4 * j + 3] + b.y;
                if (g.relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); v2 = fmaxf(v2, 0.f); v3 = fmaxf(v3, 0.f); }
                unsigned char* bx = buf + (t >> 1) * OUT_BOX_BYTES + (((t & 1) ^ sw) << 4) + q * 4;
                *reinterpret_cast<uint32_t*>(bx + r * 32) = pack_bf16(v0, v1);
                *reinterpret_cast<uint32_t*>(bx + (r + 8) * 32) = pack_bf16(v2, v3);
            }
            fence_proxy_async_shared();
            __syncwarp();
            if (lane == 0) {
                for (int x = 0; x < boxes; x++) {
                    const int n0 = n_blk * BN + p + x * OUT_BOX_COLS;
                    if (n0 >= n_lim) break;
                    if (g.mode == MODE_SCATTER) {
                        const int st = dest_s[n0 >> 4].store;
                        tma_store_2d(&maps.m[st >> 16], buf + x * OUT_BOX_BYTES, st & 0xffff, m0);
                    } else {
                        tma_store_2d(&maps.m[0], buf + x * OUT_BOX_BYTES, n0, m0);
                    }
                }
                bulk_commit();
            }
            ob ^= 1;
        }
    }
}

// ------------------------------------------------------------------ wgmma GEMM
// NG = ceil(block_n / 64) column groups: 32 * NG accumulator registers per consumer thread; the last group is LASTW
// columns wide (block_n == (NG - 1) * 64 + LASTW)
template <int NG, int LASTW>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
k_gemm_wg(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
          const __grid_constant__ CUtensorMap tmap_src, const __grid_constant__ StoreMaps smaps, GemmArgs g) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    // carve: [stages][A 16 KB | B block_n*128 B] then resident weights, pass-through tiles, staging / output chunks
    // (1024-byte aligned: everything before is a multiple of 2 KB), tables, barriers
    unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    const int a_bytes = BM * BK * 2;
    const int b_bytes = g.block_n * BK * 2;
    // weights-resident mode: the ring carries only A; the CTA's weight tile (all K blocks of ONE n block) is
    // loaded once -- weights are otherwise re-fetched from L2 for every M tile and outweigh the A traffic
    const int stage_bytes = a_bytes + (g.b_resident ? 0 : b_bytes);
    unsigned char* b_res = smem + (size_t)g.stages * stage_bytes;
    const size_t b_res_bytes = g.b_resident ? (size_t)g.num_k_blocks * b_bytes : 0;
    // pass-through tiles of the fused shuffle: [2][BM rows][block_n] bf16, filled by TMA
    const int src_bytes = g.src_tma ? BM * g.block_n * 2 : 0;
    unsigned char* src_tiles = b_res + b_res_bytes;
    // f32 staging tiles of warp_epilogue, or the bf16 output chunks of warp_epilogue_tma (same region)
    float* stg_s = reinterpret_cast<float*>(src_tiles + 2 * (size_t)src_bytes);
    float* bias_s = reinterpret_cast<float*>(reinterpret_cast<unsigned char*>(stg_s) + STG_BYTES);   // [n_blocks * block_n]
    DestGroup* dest_s = reinterpret_cast<DestGroup*>(bias_s + g.n_blocks * g.block_n);   // [n_blocks * block_n / 16]
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(dest_s + g.n_blocks * g.block_n / CHUNK);   // [stages]
    uint64_t* empty_bar = full_bar + g.stages;                          // [stages]
    uint64_t* src_full = empty_bar + g.stages;                          // [2]
    uint64_t* src_empty = src_full + 2;                                 // [2]
    uint64_t* b_full = src_empty + 2;                                   // [1]

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&tmap_a);
        tma_prefetch_desc(&tmap_b);
        if (g.src_tma) tma_prefetch_desc(&tmap_src);
    }
    for (int i = threadIdx.x; i < g.n_blocks * g.block_n; i += GEMM_THREADS) bias_s[i] = g.bias[i];
    if (g.mode == MODE_SCATTER)
        for (int i = threadIdx.x; i < g.n_blocks * g.block_n / CHUNK; i += GEMM_THREADS) dest_s[i] = g.dest[i];
    if (warp == 1 && lane == 0) {
        for (int s = 0; s < g.stages; s++) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], CONSUMER_WARPS); }
        for (int a = 0; a < 2; a++) { mbar_init(&src_full[a], 1); mbar_init(&src_empty[a], CONSUMER_WARPS); }
        mbar_init(b_full, 1);
        fence_barrier_init();
    }
    __syncthreads();
    // the resident weight tile does not depend on the predecessor kernel: its loads go out before the grid-dependency
    // wait and land while the predecessor's last CTAs drain
    if (warp == 0 && lane == 0 && g.b_resident) {
        mbar_expect_tx(b_full, (uint32_t)b_res_bytes);
        for (int kb = 0; kb < g.num_k_blocks; kb++)
            tma_load_2d(b_res + (size_t)kb * b_bytes, &tmap_b, b_full, kb * BK, (int)(blockIdx.x % g.n_blocks) * g.block_n);
    }
    pdl_launch_dependents();
    pdl_wait();

    // tile schedule: streaming mode walks (m_blk, n_blk) tiles round-robin over the CTAs; weights-resident mode
    // pins one n block per CTA (gridDim.x is a multiple of n_blocks) and walks M tiles only
    const int num_tiles = g.b_resident ? 0 : g.m_blocks * g.n_blocks;
    const int my_n = g.b_resident ? (int)(blockIdx.x % g.n_blocks) : 0;
    const int m_first = g.b_resident ? (int)(blockIdx.x / g.n_blocks) : 0;
    const int m_step = g.b_resident ? (int)(gridDim.x / g.n_blocks) : 0;
#define PIFPAF_TILE_LOOP(m_blk, n_blk)                                                                             \
    for (int it__ = g.b_resident ? m_first : (int)blockIdx.x, m_blk = 0, n_blk = 0;                                 \
         (g.b_resident ? it__ < g.m_blocks : it__ < num_tiles) &&                                                   \
         ((m_blk = g.b_resident ? it__ : it__ / g.n_blocks), (n_blk = g.b_resident ? my_n : it__ % g.n_blocks), true); \
         it__ += g.b_resident ? m_step : (int)gridDim.x)

    // 384 threads share 64 K registers: the producer warpgroup keeps 40 each, the consumers take 232 for their
    // 32 * NG accumulators and the epilogue
    if (warp < 4) {
        reg_dealloc<40>();
        // ===== TMA producer (one elected lane of warp 0) =====
        if (warp == 0 && lane == 0) {
            int stage = 0; uint32_t phase = 0;
            int sbuf = 0; uint32_t sbuf_phase = 0;
            PIFPAF_TILE_LOOP(m_blk, n_blk) {
                int cb = 0, cy = 0, cx = 0, cimg = 0;
                if (g.conv_k > 0) {
                    const int per_img = g.tiles_x * g.tiles_y;
                    cimg = m_blk / per_img;
                    const int t = m_blk - cimg * per_img;
                    cy = (t / g.tiles_x) * PH * g.conv_stride - g.conv_pad;
                    cx = (t % g.tiles_x) * PW * g.conv_stride - g.conv_pad;
                }
                for (int kb = 0; kb < g.num_k_blocks; kb++) {
                    mbar_wait(&empty_bar[stage], phase ^ 1);
                    unsigned char* sa = smem + (size_t)stage * stage_bytes;
                    unsigned char* sb = sa + a_bytes;
                    mbar_expect_tx(&full_bar[stage], (uint32_t)stage_bytes);
                    if (g.conv_k > 0) {
                        const int tap = kb / g.conv_cblocks;
                        cb = kb - tap * g.conv_cblocks;
                        tma_load_4d(sa, &tmap_a, &full_bar[stage], cb * BK, cx + (tap % g.conv_k) * g.conv_dil,
                                    cy + (tap / g.conv_k) * g.conv_dil, cimg);
                    } else {
                        tma_load_2d(sa, &tmap_a, &full_bar[stage], g.a_col0 + kb * BK, m_blk * BM);
                    }
                    if (!g.b_resident) tma_load_2d(sb, &tmap_b, &full_bar[stage], kb * BK, n_blk * g.block_n);
                    if (++stage == g.stages) { stage = 0; phase ^= 1; }
                }
                if (g.src_tma) {
                    // pass-through tile of this output tile; its buffer is free once the epilogue of the tile two
                    // tiles ago has released it
                    mbar_wait(&src_empty[sbuf], sbuf_phase ^ 1);
                    mbar_expect_tx(&src_full[sbuf], (uint32_t)src_bytes);
                    tma_load_2d(src_tiles + (size_t)sbuf * src_bytes, &tmap_src, &src_full[sbuf],
                                n_blk * g.block_n, m_blk * BM);
                    if (++sbuf == 2) { sbuf = 0; sbuf_phase ^= 1; }
                }
            }
        }
    } else {
        reg_alloc<232>();
        // ===== consumer warpgroups: rows [64 * wg, +64) of every tile =====
        const int cw = warp - 4, wg = cw >> 2;
        float acc[NG][32];
#pragma unroll
        for (int gi = 0; gi < NG; gi++)
#pragma unroll
            for (int i = 0; i < 32; i++) acc[gi][i] = 0.f;
        float* stg = stg_s + cw * 16 * STG_LD;
        unsigned char* obuf = reinterpret_cast<unsigned char*>(stg_s) + cw * OUT_WARP_BYTES;
        int ob = 0;
        int stage = 0; uint32_t phase = 0;
        int sbuf = 0; uint32_t sbuf_phase = 0;
        if (g.b_resident) mbar_wait(b_full, 0);
        PIFPAF_TILE_LOOP(m_blk, n_blk) {
            int prev = 0;
            for (int kb = 0; kb < g.num_k_blocks; kb++) {
                mbar_wait(&full_bar[stage], phase);
                const uint32_t sa = smem_u32(smem + (size_t)stage * stage_bytes);
                const uint32_t sb = g.b_resident ? smem_u32(b_res + (size_t)kb * b_bytes) : sa + a_bytes;
#pragma unroll
                for (int gi = 0; gi < NG; gi++) fence_acc(acc[gi]);
                wgmma_fence();
                mma_k_block<NG, LASTW>(acc, sa + wg * WG_ROWS * BK * 2, sb, kb == 0);
                wgmma_commit();
                // the MMAs of the previous K block have retired: its slot goes back to the producer
                if (kb > 0) {
                    wgmma_wait<1>();
                    if (lane == 0) mbar_arrive(&empty_bar[prev]);
                }
                prev = stage;
                if (++stage == g.stages) { stage = 0; phase ^= 1; }
            }
            wgmma_wait<0>();
#pragma unroll
            for (int gi = 0; gi < NG; gi++) fence_acc(acc[gi]);
            if (lane == 0) mbar_arrive(&empty_bar[prev]);
            if (g.tma_store) {
                warp_epilogue_tma<NG, LASTW>(g, smaps, acc, obuf, ob, m_blk, n_blk, wg * WG_ROWS + (cw & 3) * 16,
                                             bias_s, dest_s);
                continue;
            }
            if (g.src_tma) mbar_wait(&src_full[sbuf], sbuf_phase);
            warp_epilogue<NG>(g, acc, stg, m_blk, n_blk, wg * WG_ROWS + (cw & 3) * 16, bias_s,
                              g.src_tma ? reinterpret_cast<const __nv_bfloat16*>(src_tiles + (size_t)sbuf * src_bytes) : nullptr,
                              dest_s);
            if (g.src_tma) {
                __syncwarp();
                if (lane == 0) mbar_arrive(&src_empty[sbuf]);
                if (++sbuf == 2) { sbuf = 0; sbuf_phase ^= 1; }
            }
        }
        // the dependent kernel's grid-dependency wait covers completed writes only: the tensor stores must be done
        // before this CTA exits
        if (g.tma_store && lane == 0) bulk_wait_all();
    }
}

// ------------------------------------------------------------------ SIMT debug GEMM (tests only)
// One warp per 32 rows x CHUNK columns; same epilogue as the tensor-core kernel.
__global__ void __launch_bounds__(128) k_gemm_simt(GemmArgs g) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int n_chunks = g.n_blocks * g.block_n / CHUNK;
    const long long total = (long long)g.m_blocks * 4 * n_chunks;        // 4 row quarters per M tile
    for (long long job = (long long)blockIdx.x * 4 + warp; job < total; job += (long long)gridDim.x * 4) {
        const int ch = (int)(job % n_chunks);
        const int mq = (int)(job / n_chunks);
        const int m_blk = mq >> 2, row = (mq & 3) * 32 + lane;
        const int n0 = ch * CHUNK;
        const int m = tile_row_to_m(g, m_blk, row);
        float acc[CHUNK];
#pragma unroll
        for (int j = 0; j < CHUNK; j++) acc[j] = 0.f;
        if (m >= 0) {
            if (g.conv_k == 0) {
                for (int k = 0; k < g.K; k++) {
                    const float a = __bfloat162float(g.a[(size_t)m * g.lda + k]);
#pragma unroll
                    for (int j = 0; j < CHUNK; j++) {
                        const int n = n0 + j;
                        const float wv = (n < g.N) ? __bfloat162float(g.wgt[(size_t)n * g.ldw + k]) : 0.f;
                        acc[j] = fmaf(a, wv, acc[j]);
                    }
                }
            } else {
                const int ox = m % g.Wo, oy = (m / g.Wo) % g.Ho, b = m / (g.Wo * g.Ho);
                for (int tap = 0; tap < g.conv_k * g.conv_k; tap++) {
                    const int iy = oy * g.conv_stride - g.conv_pad + (tap / g.conv_k) * g.conv_dil;
                    const int ix = ox * g.conv_stride - g.conv_pad + (tap % g.conv_k) * g.conv_dil;
                    if (iy < 0 || iy >= g.Hi || ix < 0 || ix >= g.Wi) continue;
                    const __nv_bfloat16* ap = g.a + ((size_t)(b * g.Hi + iy) * g.Wi + ix) * g.lda;
                    for (int k = 0; k < g.K; k++) {
                        const float a = __bfloat162float(ap[k]);
#pragma unroll
                        for (int j = 0; j < CHUNK; j++) {
                            const int n = n0 + j;
                            const float wv = (n < g.N)
                                ? __bfloat162float(g.wgt[(size_t)n * g.ldw + (size_t)tap * g.conv_cblocks * BK + k]) : 0.f;
                            acc[j] = fmaf(a, wv, acc[j]);
                        }
                    }
                }
            }
        }
        if (n0 < ((g.N + 7) & ~7)) epilogue_chunk(g, m, n0, acc, g.bias + n0, nullptr, g.dest);
    }
}

// ------------------------------------------------------------------ depthwise kxk conv, NHWC bf16
// one thread: one output pixel x 8 channels (16-byte vectors); weights [k*k][C8*8] f32, bias [C]
struct DwArgs {
    const __nv_bfloat16* in; int ld_in; int in_col_off;
    __nv_bfloat16* out; int ld_out; int out_col_off;
    const float* weight; const float* bias;
    int B, Hin, Win, Hout, Wout, C8, kernel, stride, pad, relu;
};

// bf16x2 word -> two floats (bf16 -> f32 is a 16-bit shift)
__device__ __forceinline__ void unpack8(const uint4& v, float* f) {
    f[0] = __uint_as_float(v.x << 16); f[1] = __uint_as_float(v.x & 0xffff0000u);
    f[2] = __uint_as_float(v.y << 16); f[3] = __uint_as_float(v.y & 0xffff0000u);
    f[4] = __uint_as_float(v.z << 16); f[5] = __uint_as_float(v.z & 0xffff0000u);
    f[6] = __uint_as_float(v.w << 16); f[7] = __uint_as_float(v.w & 0xffff0000u);
}

// Register-tiled depthwise 5x5: one thread = 8 channels x DW_OX consecutive output pixels of one row.
// Each input vector is loaded once and feeds every output/tap it touches; the 5x8 weights of a kernel row
// stay in registers.  f32 accumulate.  (k == 5 only; other kernels take the generic path below.)
constexpr int DW_OX = 4;
constexpr int DW_OY = 8;

template <int S>
__global__ void __launch_bounds__(256) k_dwconv5(DwArgs a) {
    constexpr int NCOL = (DW_OX - 1) * S + 5;
    const int strips = (a.Wout + DW_OX - 1) / DW_OX;
    const int ytiles = (a.Hout + DW_OY - 1) / DW_OY;
    const long long total = (long long)a.B * ytiles * strips * DW_OY * a.C8;
    const int C = a.C8 * 8;
    // thread order: channels fastest (coalesced 16-byte vectors), then DW_OY vertically adjacent rows of the
    // same strip (their 5-row input windows overlap -> L1 hits), then strips, row tiles, images
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total;
         t += (long long)gridDim.x * blockDim.x) {
        const int c8 = (int)(t % a.C8);
        long long p = t / a.C8;
        const int yl = (int)(p % DW_OY); p /= DW_OY;
        const int sx = (int)(p % strips); p /= strips;
        const int oy = (int)(p % ytiles) * DW_OY + yl;
        const int b = (int)(p / ytiles);
        if (oy >= a.Hout) continue;
        const int ox0 = sx * DW_OX;
        const int ix0 = ox0 * S - a.pad;
        float acc[DW_OX][8];
        {
            const float4 b0 = __ldg(reinterpret_cast<const float4*>(a.bias + c8 * 8));
            const float4 b1 = __ldg(reinterpret_cast<const float4*>(a.bias + c8 * 8 + 4));
#pragma unroll
            for (int o = 0; o < DW_OX; o++) {
                acc[o][0] = b0.x; acc[o][1] = b0.y; acc[o][2] = b0.z; acc[o][3] = b0.w;
                acc[o][4] = b1.x; acc[o][5] = b1.y; acc[o][6] = b1.z; acc[o][7] = b1.w;
            }
        }
#pragma unroll
        for (int ky = 0; ky < 5; ky++) {
            const int iy = oy * S - a.pad + ky;
            if (iy < 0 || iy >= a.Hin) continue;
            float w[5][8];
#pragma unroll
            for (int kx = 0; kx < 5; kx++) {
                const float* wp = a.weight + (size_t)(ky * 5 + kx) * C + c8 * 8;
                const float4 w0 = __ldg(reinterpret_cast<const float4*>(wp));
                const float4 w1 = __ldg(reinterpret_cast<const float4*>(wp + 4));
                w[kx][0] = w0.x; w[kx][1] = w0.y; w[kx][2] = w0.z; w[kx][3] = w0.w;
                w[kx][4] = w1.x; w[kx][5] = w1.y; w[kx][6] = w1.z; w[kx][7] = w1.w;
            }
            const __nv_bfloat16* rowp = a.in + ((size_t)(b * a.Hin + iy) * a.Win) * a.ld_in + a.in_col_off + c8 * 8;
#pragma unroll
            for (int col = 0; col < NCOL; col++) {
                const int ix = ix0 + col;
                if (ix < 0 || ix >= a.Win) continue;
                const uint4 v = __ldg(reinterpret_cast<const uint4*>(rowp + (size_t)ix * a.ld_in));
                float f[8];
                unpack8(v, f);
#pragma unroll
                for (int o = 0; o < DW_OX; o++) {
                    const int kx = col - o * S;       // compile-time after unrolling
                    if (kx < 0 || kx >= 5) continue;
#pragma unroll
                    for (int j = 0; j < 8; j++) acc[o][j] = fmaf(f[j], w[kx][j], acc[o][j]);
                }
            }
        }
#pragma unroll
        for (int o = 0; o < DW_OX; o++) {
            const int ox = ox0 + o;
            if (ox >= a.Wout) continue;
#pragma unroll
            for (int j = 0; j < 8; j++) acc[o][j] = act_f(acc[o][j], a.relu);
            uint4 ov;
            ov.x = pack_bf16(acc[o][0], acc[o][1]); ov.y = pack_bf16(acc[o][2], acc[o][3]);
            ov.z = pack_bf16(acc[o][4], acc[o][5]); ov.w = pack_bf16(acc[o][6], acc[o][7]);
            *reinterpret_cast<uint4*>(a.out + ((size_t)(b * a.Hout + oy) * a.Wout + ox) * a.ld_out + a.out_col_off + c8 * 8) = ov;
        }
    }
}

// Depthwise KS x KS (5x5: ShuffleNetV2K, also with taps D = 2 pixels apart; 3x3: MobileNetV2) with TMA-staged input
// tiles.  A persistent CTA walks (channel block, image, tile) work items; the input window of an item
// ((TH-1)*S+(KS-1)*D+1 x (TW-1)*S+(KS-1)*D+1 pixels x 64 channels, 4-D tensor map, out-of-bounds zero fill
// == the conv padding) is streamed by TMA into an NSTAGE-deep shared-memory ring.  There is no CTA-wide barrier in
// the steady state: every warp counts itself out of a ring slot with one shared-memory atomic, and the warp that
// finishes a slot LAST re-arms it with the TMA of the item NSTAGE rounds ahead, so fast warps (edge tiles with
// out-of-range blocks) run ahead of slow ones by up to NSTAGE-1 items.
// Compute mapping (register blocking in BOTH spatial directions): one warp = one 4 x BW block of output pixels,
// one lane = one channel pair.  The lane keeps its KS*KS x 2 weights and a 4 x BW x 2 f32 accumulator in registers and
// reads every input pixel of the block's window exactly once (4 bytes per lane, 128 bytes per warp request: one
// conflict-free wavefront).
template <int S, int TH, int TW, int BW, int NSTAGE, int KS = 5, int D = 1>
struct DwTile {
    static constexpr int IH = (TH - 1) * S + (KS - 1) * D + 1, IW = (TW - 1) * S + (KS - 1) * D + 1;
    static constexpr int BYTES = IH * IW * 64 * 2;
    static constexpr int WARPS = (TH / 4) * (TW / BW);
    static constexpr int THREADS = WARPS * 32;
    static constexpr int WIN_Y = 3 * S + (KS - 1) * D + 1;           // input window of a 4 x BW output block
    static constexpr int WIN_X = (BW - 1) * S + (KS - 1) * D + 1;
    static constexpr int SMEM = NSTAGE * BYTES + 128;
};

// position of a work item and its increment per persistent-loop step, kept as mixed-radix digits
// (channel block, image, tile row, tile column) so that the loop needs no integer division
struct DwPos { int c, b, y, x; };

__device__ __forceinline__ DwPos dw_decompose(int w, int per_c, int tiles_y, int tiles_x) {
    DwPos p;
    p.c = w / per_c; int r = w - p.c * per_c;
    p.b = r / (tiles_y * tiles_x); r -= p.b * tiles_y * tiles_x;
    p.y = r / tiles_x; p.x = r - p.y * tiles_x;
    return p;
}

__device__ __forceinline__ void dw_advance(DwPos& p, const DwPos& d, int B, int tiles_y, int tiles_x) {
    p.x += d.x; int carry = p.x >= tiles_x; p.x -= carry ? tiles_x : 0;
    p.y += d.y + carry; carry = p.y >= tiles_y; p.y -= carry ? tiles_y : 0;
    p.b += d.b + carry; carry = p.b >= B; p.b -= carry ? B : 0;
    p.c += d.c + carry;
}

// channel-block-FASTEST item order (CBF): item = (image, tile row, tile column, channel block) with the channel block
// as the fastest digit, so the 128-byte channel blocks of one pixel (352 / 704-byte pixels: most blocks straddle a
// 64-byte DRAM atom) and the halos of neighbouring tiles are fetched by CTAs running at the same time and meet in L2.
__device__ __forceinline__ DwPos dw_decompose_cf(int w, int cblks, int tiles_y, int tiles_x) {
    DwPos p;
    p.c = w % cblks; int r = w / cblks;
    p.x = r % tiles_x; r /= tiles_x;
    p.y = r % tiles_y; p.b = r / tiles_y;
    return p;
}

__device__ __forceinline__ void dw_advance_cf(DwPos& p, const DwPos& d, int cblks, int tiles_y, int tiles_x) {
    p.c += d.c; int carry = p.c >= cblks; p.c -= carry ? cblks : 0;
    p.x += d.x + carry; carry = p.x >= tiles_x; p.x -= carry ? tiles_x : 0;
    p.y += d.y + carry; carry = p.y >= tiles_y; p.y -= carry ? tiles_y : 0;
    p.b += d.b + carry;
}

// One warp's share of a depthwise KS x KS item (KS = 5 or 3; taps D pixels apart): the 4 x BW output pixels at
// (oy0, ox0) of image b, lane = the channel pair c0, c0 + 1; bias initialises the f32 sums, the KS * KS taps run in
// (ky, kx) order (the order of k_dwconv, so the 3x3 and dilated results equal its bit for bit), activation a.relu,
// bf16 stores.  Tap (ky, kx) of output (i, j) reads window row i * S + ky * D, column j * S + kx * D.
// win: the item's input window in shared memory, IW pixels per row, 128 bytes (64 channels) per pixel; p0: the
// window pixel at the block's first tap.  SWZ: the 16-byte units of pixel p sit at unit ^ (p & 7) (k_pw_dw's
// intermediate window, which its wgmma epilogue writes without bank conflicts that way); the eight possible units
// are resolved once per block, so the loads need no address arithmetic.
template <int S, int BW, int IW, bool SWZ, int KS = 5, int D = 1>
__device__ __forceinline__ void dw5_block(const DwArgs& a, const unsigned char* win, int p0, int lane,
                                          const float (&wgt)[KS * KS][2], float bias0, float bias1, int b, int oy0,
                                          int ox0, int c0) {
    constexpr int WIN_Y = 3 * S + (KS - 1) * D + 1, WIN_X = (BW - 1) * S + (KS - 1) * D + 1;
    const unsigned char* tile = win + p0 * 128 + (SWZ ? (lane & 3) * 4 : lane * 4);
    const unsigned char* rows[SWZ ? 8 : 1];          // SWZ: the lane's word in a pixel p with p & 7 == c
#pragma unroll
    for (int c = 0; c < (SWZ ? 8 : 1); c++) rows[c] = tile + (SWZ ? ((lane >> 2) ^ ((p0 + c) & 7)) << 4 : 0);
    float acc[4][BW][2];
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < BW; j++) { acc[i][j][0] = bias0; acc[i][j][1] = bias1; }
#pragma unroll
    for (int ry = 0; ry < WIN_Y; ry++) {
        float f[WIN_X][2];
#pragma unroll
        for (int cx = 0; cx < WIN_X; cx++) {
            const int p = ry * IW + cx;
            const uint32_t v = *reinterpret_cast<const uint32_t*>(rows[SWZ ? p & 7 : 0] + p * 128);
            f[cx][0] = __uint_as_float(v << 16);
            f[cx][1] = __uint_as_float(v & 0xffff0000u);
        }
#pragma unroll
        for (int i = 0; i < 4; i++) {
            const int dy = ry - i * S;                    // compile-time after unrolling
            if (dy < 0 || dy % D != 0 || dy / D >= KS) continue;
            const int ky = dy / D;
#pragma unroll
            for (int kx = 0; kx < KS; kx++) {
#pragma unroll
                for (int j = 0; j < BW; j++) {
                    acc[i][j][0] = fmaf(f[j * S + kx * D][0], wgt[ky * KS + kx][0], acc[i][j][0]);
                    acc[i][j][1] = fmaf(f[j * S + kx * D][1], wgt[ky * KS + kx][1], acc[i][j][1]);
                }
            }
        }
    }
    if (a.relu) {
#pragma unroll
        for (int i = 0; i < 4; i++)
#pragma unroll
            for (int j = 0; j < BW; j++) {
                acc[i][j][0] = fmaxf(acc[i][j][0], 0.f); acc[i][j][1] = fmaxf(acc[i][j][1], 0.f);
            }
    }
    // ReLU6 is compiled into the 3x3 instantiations only: any change to the epilogue moves the register allocation of
    // the 5x5 ones (k_dwconv5_tma and k_pw_dw), so a 5x5 depthwise conv with ReLU6 -- no network has one -- runs
    // k_dwconv5 (pifpaf_net_dwconv)
    if constexpr (KS == 3) {
        if (a.relu == ACT_RELU6) {
#pragma unroll
            for (int i = 0; i < 4; i++)
#pragma unroll
                for (int j = 0; j < BW; j++) {
                    acc[i][j][0] = fminf(acc[i][j][0], 6.f); acc[i][j][1] = fminf(acc[i][j][1], 6.f);
                }
        }
    }
    const size_t out_row = (size_t)a.Wout * a.ld_out;           // elements per output image row
    __nv_bfloat16* orow = a.out + ((size_t)(b * a.Hout + oy0) * a.Wout + ox0) * a.ld_out + a.out_col_off + c0;
    if (oy0 + 4 <= a.Hout && ox0 + BW <= a.Wout) {          // interior block: no per-pixel predicates
#pragma unroll
        for (int i = 0; i < 4; i++) {
            __nv_bfloat16* op = orow + i * out_row;
#pragma unroll
            for (int j = 0; j < BW; j++)
                *reinterpret_cast<uint32_t*>(op + (size_t)j * a.ld_out) = pack_bf16(acc[i][j][0], acc[i][j][1]);
        }
    } else {
#pragma unroll
        for (int i = 0; i < 4; i++) {
            if (oy0 + i >= a.Hout) continue;
            __nv_bfloat16* op = orow + i * out_row;
#pragma unroll
            for (int j = 0; j < BW; j++) {
                if (ox0 + j >= a.Wout) continue;
                *reinterpret_cast<uint32_t*>(op + (size_t)j * a.ld_out) = pack_bf16(acc[i][j][0], acc[i][j][1]);
            }
        }
    }
}

template <int S, int TH, int TW, int BW, int NSTAGE, bool CBF = false, int KS = 5, int D = 1>
__global__ void __launch_bounds__(DwTile<S, TH, TW, BW, NSTAGE, KS, D>::THREADS, 2)
k_dwconv5_tma(const __grid_constant__ CUtensorMap tmap_in, DwArgs a) {
    using T = DwTile<S, TH, TW, BW, NSTAGE, KS, D>;
    constexpr int TAPS = KS * KS;
    extern __shared__ __align__(128) unsigned char dsm_raw[];
    // align inside the shared window with pointer arithmetic on the array itself (keeps the address space known to
    // the compiler: LDS instead of generic loads)
    unsigned char* dsm = dsm_raw + ((128u - (smem_u32(dsm_raw) & 127u)) & 127u);
    __shared__ uint64_t full[NSTAGE];
    __shared__ int done[NSTAGE];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int tiles_x = (a.Wout + TW - 1) / TW, tiles_y = (a.Hout + TH - 1) / TH;
    const int cblks = (a.C8 + 7) / 8;
    const int per_c = a.B * tiles_y * tiles_x;
    const int total = per_c * cblks;
    const int C = a.C8 * 8;
    // CBF: the channel block changes with (almost) every item, so the weights [TAPS][C] + bias [C] are staged in
    // shared memory once per CTA and re-read from there (TAPS + 1 LDS.64 per item)
    const float* s_w = reinterpret_cast<const float*>(dsm + (size_t)NSTAGE * T::BYTES);
    if (CBF) {
        float* sw = reinterpret_cast<float*>(dsm + (size_t)NSTAGE * T::BYTES);
        for (int i = tid; i < TAPS * C; i += T::THREADS) sw[i] = a.weight[i];
        for (int i = tid; i < C; i += T::THREADS) sw[TAPS * C + i] = a.bias[i];
    }
    auto decompose = [&](int w) { return CBF ? dw_decompose_cf(w, cblks, tiles_y, tiles_x) : dw_decompose(w, per_c, tiles_y, tiles_x); };
    auto advance = [&](DwPos& p, const DwPos& d) {
        if (CBF) dw_advance_cf(p, d, cblks, tiles_y, tiles_x); else dw_advance(p, d, a.B, tiles_y, tiles_x);
    };

    auto issue = [&](const DwPos& p, int buf) {
        mbar_expect_tx(&full[buf], (uint32_t)T::BYTES);
        tma_load_4d(dsm + (size_t)buf * T::BYTES, &tmap_in, &full[buf], p.c * 64, p.x * TW * S - a.pad,
                    p.y * TH * S - a.pad, p.b);
    };

    pdl_launch_dependents();
    pdl_wait();
    if (tid == 0) {
#pragma unroll
        for (int s = 0; s < NSTAGE; s++) { mbar_init(&full[s], 1); done[s] = 0; }
        fence_barrier_init();
        tma_prefetch_desc(&tmap_in);
#pragma unroll
        for (int s = 0; s < NSTAGE; s++) {
            const int w0 = blockIdx.x + s * gridDim.x;
            if (w0 < total) issue(decompose(w0), s);
        }
    }
    __syncthreads();

    const int by = warp / (TW / BW), bx = warp % (TW / BW);     // 4 x BW output block of this warp inside the tile
    const DwPos step = decompose(gridDim.x);
    const DwPos step_ring = decompose(NSTAGE * gridDim.x);
    DwPos pos = decompose(blockIdx.x);
    int buf = 0; uint32_t phase = 0;
    int w_cblk = -1;
    float wgt[TAPS][2];
    float bias0 = 0.f, bias1 = 0.f;
    for (int w = blockIdx.x; w < total; w += gridDim.x) {
        const int c0 = pos.c * 64 + lane * 2;
        if (pos.c != w_cblk) {                      // (re)load this lane's weights: rarely, the block index is slowest
            w_cblk = pos.c;
            const bool cok = c0 < C;
#pragma unroll
            for (int tp = 0; tp < TAPS; tp++) {
                const float2 wv = !cok ? make_float2(0.f, 0.f)
                                  : CBF ? *reinterpret_cast<const float2*>(s_w + (size_t)tp * C + c0)
                                        : __ldg(reinterpret_cast<const float2*>(a.weight + (size_t)tp * C + c0));
                wgt[tp][0] = wv.x; wgt[tp][1] = wv.y;
            }
            const float2 bv = !cok ? make_float2(0.f, 0.f)
                              : CBF ? *reinterpret_cast<const float2*>(s_w + TAPS * (size_t)C + c0)
                                    : __ldg(reinterpret_cast<const float2*>(a.bias + c0));
            bias0 = bv.x; bias1 = bv.y;
        }
        const int oy0 = pos.y * TH + by * 4, ox0 = pos.x * TW + bx * BW;
        // every warp waits (also those whose block lies past the image edge): passing this wait proves that all
        // warps counted out of the slot's previous item, so the per-slot count never mixes two items
        mbar_wait(&full[buf], phase);
        if (oy0 < a.Hout && ox0 < a.Wout && c0 < C)
            dw5_block<S, BW, T::IW, false, KS, D>(a, dsm + (size_t)buf * T::BYTES, (by * 4 * S) * T::IW + bx * BW * S,
                                               lane, wgt, bias0, bias1, pos.b, oy0, ox0, c0);
        // count this warp out of the slot; the last one out re-arms it.  Every shared-memory read of the slot has
        // been consumed by an fma above (results are in registers), the fence orders them before the count.
        __syncwarp();
        if (lane == 0) {
            __threadfence_block();
            if (atomicAdd(&done[buf], 1) == T::WARPS - 1) {
                done[buf] = 0;
                if (w + NSTAGE * (int)gridDim.x < total) {
                    DwPos pn = pos;
                    advance(pn, step_ring);
                    issue(pn, buf);
                }
            }
        }
        advance(pos, step);
        if (++buf == NSTAGE) { buf = 0; phase ^= 1; }
    }
}

// tile shapes: stride 1 -> 8x16 outputs, 4x4 blocks (8 warps, 30 KB window, 3-deep ring, 2 CTAs per SM);
//              stride 2 -> 8x16 outputs, 4x4 blocks (8 warps, 85 KB window, 2-deep ring, 1 CTA per SM): the
//              stride-2 launches are DRAM-bound on halo re-reads, the wide tile has the smaller halo (1.30x
//              against 1.41x for 8x8)
// 3x3: the same tiles and blocks; the smaller windows buy one more ring slot at the same bytes in flight per SM:
//              stride 1 -> 23 KB window, 4-deep ring, 2 CTAs per SM; stride 2 -> 72 KB window, 3-deep ring, 1 CTA per SM
// 5x5 with dilation 2 (stride 1; ShuffleNetV2K stage 4 under --shufflenetv2k-stage4-dilation 2): the stride-1 tile
//              and blocks with a 16 x 24 pixel window (48 KB; a 12 x 12 window per 4 x 4 block); 2-deep ring, 2 CTAs
//              per SM (192 KB of windows per SM, 16 warps as DwS1).  A 3-deep ring would leave one CTA per SM.
constexpr int DW1_TH = 8, DW1_TW = 16, DW2_TH = 8, DW2_TW = 16;
using DwS1 = DwTile<1, DW1_TH, DW1_TW, 4, 3>;
using DwS1D2 = DwTile<1, DW1_TH, DW1_TW, 4, 2, 5, 2>;
using DwS2 = DwTile<2, DW2_TH, DW2_TW, 4, 2>;
using DwS1K3 = DwTile<1, DW1_TH, DW1_TW, 4, 4, 3>;
using DwS2K3 = DwTile<2, DW2_TH, DW2_TW, 4, 3, 3>;

// 3x3 max pool, pad 1, stride a.stride (torchvision's MaxPool2d(3, 2, 1) in the ResNet input block,
// basenetworks.py:85-93): one output pixel x 8 channels (one 16-byte vector) per thread.  Taps outside the image are
// skipped, as torch's -inf padding does; the centre tap is always inside.  The weight / bias fields of DwArgs are unused.
__global__ void __launch_bounds__(256) k_maxpool(DwArgs a) {
    pdl_launch_dependents();
    pdl_wait();
    const long long total = (long long)a.B * a.Hout * a.Wout * a.C8;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total;
         t += (long long)gridDim.x * blockDim.x) {
        const int c8 = (int)(t % a.C8);
        long long p = t / a.C8;
        const int ox = (int)(p % a.Wout); p /= a.Wout;
        const int oy = (int)(p % a.Hout);
        const int b = (int)(p / a.Hout);
        const __nv_bfloat162 ninf = __bfloat162bfloat162(__ushort_as_bfloat16((unsigned short)0xff80u));
        __nv_bfloat162 m[4] = {ninf, ninf, ninf, ninf};
#pragma unroll
        for (int ky = 0; ky < 3; ky++) {
            const int iy = oy * a.stride - 1 + ky;
            if (iy < 0 || iy >= a.Hin) continue;
#pragma unroll
            for (int kx = 0; kx < 3; kx++) {
                const int ix = ox * a.stride - 1 + kx;
                if (ix < 0 || ix >= a.Win) continue;
                const uint4 v = __ldg(reinterpret_cast<const uint4*>(
                    a.in + ((size_t)(b * a.Hin + iy) * a.Win + ix) * a.ld_in + a.in_col_off + c8 * 8));
                const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
                for (int j = 0; j < 4; j++) m[j] = __hmax2(m[j], h[j]);
            }
        }
        *reinterpret_cast<uint4*>(a.out + ((size_t)(b * a.Hout + oy) * a.Wout + ox) * a.ld_out + a.out_col_off + c8 * 8) =
            *reinterpret_cast<const uint4*>(m);
    }
}

// generic depthwise kxk (any kernel / stride / dilation): one output pixel x 8 channels per thread.  The dilation is
// a parameter of its own: a DwArgs field would move the layout of PwDwArgs (which embeds DwArgs) and with it the
// register allocation of k_pw_dw
__global__ void __launch_bounds__(256) k_dwconv(DwArgs a, int dil) {
    const long long total = (long long)a.B * a.Hout * a.Wout * a.C8;
    const int C = a.C8 * 8;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total;
         t += (long long)gridDim.x * blockDim.x) {
        const int c8 = (int)(t % a.C8);
        long long p = t / a.C8;
        const int ox = (int)(p % a.Wout); p /= a.Wout;
        const int oy = (int)(p % a.Hout);
        const int b = (int)(p / a.Hout);
        float acc[8];
        const float4 b0 = *reinterpret_cast<const float4*>(a.bias + c8 * 8);
        const float4 b1 = *reinterpret_cast<const float4*>(a.bias + c8 * 8 + 4);
        acc[0] = b0.x; acc[1] = b0.y; acc[2] = b0.z; acc[3] = b0.w;
        acc[4] = b1.x; acc[5] = b1.y; acc[6] = b1.z; acc[7] = b1.w;
        for (int ky = 0; ky < a.kernel; ky++) {
            const int iy = oy * a.stride - a.pad + ky * dil;
            if (iy < 0 || iy >= a.Hin) continue;
            for (int kx = 0; kx < a.kernel; kx++) {
                const int ix = ox * a.stride - a.pad + kx * dil;
                if (ix < 0 || ix >= a.Win) continue;
                const uint4 v = __ldg(reinterpret_cast<const uint4*>(
                    a.in + ((size_t)(b * a.Hin + iy) * a.Win + ix) * a.ld_in + a.in_col_off + c8 * 8));
                const float* wp = a.weight + (size_t)(ky * a.kernel + kx) * C + c8 * 8;
                const float4 w0 = __ldg(reinterpret_cast<const float4*>(wp));
                const float4 w1 = __ldg(reinterpret_cast<const float4*>(wp + 4));
                const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
                const float2 f0 = __bfloat1622float2(h[0]), f1 = __bfloat1622float2(h[1]);
                const float2 f2 = __bfloat1622float2(h[2]), f3 = __bfloat1622float2(h[3]);
                acc[0] = fmaf(f0.x, w0.x, acc[0]); acc[1] = fmaf(f0.y, w0.y, acc[1]);
                acc[2] = fmaf(f1.x, w0.z, acc[2]); acc[3] = fmaf(f1.y, w0.w, acc[3]);
                acc[4] = fmaf(f2.x, w1.x, acc[4]); acc[5] = fmaf(f2.y, w1.y, acc[5]);
                acc[6] = fmaf(f3.x, w1.z, acc[6]); acc[7] = fmaf(f3.y, w1.w, acc[7]);
            }
        }
#pragma unroll
        for (int j = 0; j < 8; j++) acc[j] = act_f(acc[j], a.relu);
        uint4 o;
        o.x = pack_bf16(acc[0], acc[1]); o.y = pack_bf16(acc[2], acc[3]);
        o.z = pack_bf16(acc[4], acc[5]); o.w = pack_bf16(acc[6], acc[7]);
        *reinterpret_cast<uint4*>(a.out + ((size_t)(b * a.Hout + oy) * a.Wout + ox) * a.ld_out + a.out_col_off + c8 * 8) = o;
    }
}

// ------------------------------------------------------------------ fused depthwise 5x5 -> 1x1 GEMM
// InvertedResidualK branch2 tail (basenetworks.py:219-226: dw5x5, BN, 1x1, BN, ReLU) as ONE kernel: the depthwise
// output never visits HBM.  Per CTA (persistent over 8 x 16 output-pixel patches == 128-row M tiles), per 64-channel
// K block:
//   warp 8     TMA producer: the patch's input window (12 x 20 pixels x 64 channels, zero fill == conv padding) into
//              a window ring, and the K block of this CTA's 1x1 weights [block_n x 64] into a B ring
//   warps 0-7  two warpgroups, each owning 64 rows (4 x 16 pixels) of the patch.  Depthwise: one warp = a 4 x 4 block
//              of output pixels, one lane = a channel pair (the register-blocked FMA loop of k_dwconv5_tma); results
//              go as bf16 straight into the 128B-swizzled K-major A stage (row = pixel of the patch, the layout TMA
//              would have produced), fence.proxy.async + a warpgroup barrier, then wgmma.mma_async of the warpgroup's
//              own 64 rows.  The MMAs of K block kb run under the depthwise FMAs of K block kb + 1 (same warps: the
//              tensor core works while they compute), so one A stage is enough.  Epilogue as in k_gemm_wg.
// The accumulator lives in registers beside the depthwise working set: block_n <= 192 columns per CTA (NG <= 3).
// Wider outputs take n_blocks CTAs per patch, each recomputing the depthwise sums for its own column block.
constexpr int FD_THREADS = 32 * (CONSUMER_WARPS + 1);     // 288
constexpr int FD_MAX_BLOCK_N = 3 * NGROUP;

struct FusedArgs {
    const float* dw_weight;      // [25][C] f32, tap-major
    const float* dw_bias;        // [C]
    int C;                       // physical channels of the depthwise input (multiple of 8)
    int dw_relu, pad;
    int ws, bs;                  // ring depths: windows, B stages
};

template <int S, int NG, int LASTW>
__global__ void __launch_bounds__(FD_THREADS, 1)
k_dw_gemm(const __grid_constant__ CUtensorMap tmap_win, const __grid_constant__ CUtensorMap tmap_b, GemmArgs g, FusedArgs f) {
    using T = DwTile<S, PH, PW, 4, 1>;
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    const int a_bytes = BM * BK * 2;                     // 16 KB
    const int b_bytes = g.block_n * BK * 2;              // multiple of 1024 (block_n % 16 == 0)
    const int n_pad = g.block_n * g.n_blocks;
    unsigned char* a_st = smem;
    unsigned char* b_st = a_st + a_bytes;
    unsigned char* win = b_st + (size_t)f.bs * b_bytes;
    float* bias_s = reinterpret_cast<float*>(win + (size_t)f.ws * T::BYTES);
    DestGroup* dest_s = reinterpret_cast<DestGroup*>(bias_s + n_pad);
    // depthwise weights [25][C] + bias [C], staged once per CTA (a per-K-block reload from global memory would put the
    // depthwise warps on the long scoreboard: the L1 is carved down to a few KB)
    float* dww_s = reinterpret_cast<float*>(dest_s + n_pad / CHUNK);
    float* stg_s = dww_s + 26 * (size_t)f.C;
    uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<unsigned char*>(stg_s) + STG_BYTES);
    uint64_t* win_full = bars;                 uint64_t* win_empty = win_full + f.ws;
    uint64_t* b_full = win_empty + f.ws;       uint64_t* b_empty = b_full + f.bs;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (warp == CONSUMER_WARPS && lane == 0) { tma_prefetch_desc(&tmap_win); tma_prefetch_desc(&tmap_b); }
    for (int i = threadIdx.x; i < n_pad; i += FD_THREADS) bias_s[i] = g.bias[i];
    if (g.mode == MODE_SCATTER)
        for (int i = threadIdx.x; i < n_pad / CHUNK; i += FD_THREADS) dest_s[i] = g.dest[i];
    for (int i = threadIdx.x; i < 25 * f.C; i += FD_THREADS) dww_s[i] = f.dw_weight[i];
    for (int i = threadIdx.x; i < f.C; i += FD_THREADS) dww_s[25 * f.C + i] = f.dw_bias[i];
    if (warp == 0 && lane == 0) {
        for (int i = 0; i < f.ws; i++) { mbar_init(&win_full[i], 1); mbar_init(&win_empty[i], CONSUMER_WARPS); }
        for (int i = 0; i < f.bs; i++) { mbar_init(&b_full[i], 1); mbar_init(&b_empty[i], CONSUMER_WARPS); }
        fence_barrier_init();
    }
    __syncthreads();
    pdl_launch_dependents();
    pdl_wait();
    const int per_img = g.tiles_x * g.tiles_y;
    const int nkb = g.num_k_blocks;
    // one column block per CTA (gridDim.x is a multiple of n_blocks), patches round-robin
    const int n_blk = (int)(blockIdx.x % g.n_blocks);
    const int tile0 = (int)(blockIdx.x / g.n_blocks), tile_step = (int)(gridDim.x / g.n_blocks);

    if (warp == CONSUMER_WARPS) {
        // ===== TMA producer =====
        if (lane == 0) {
            int wi = 0; uint32_t wph = 0; int bi = 0; uint32_t bph = 0;
            for (int tile = tile0; tile < g.m_blocks; tile += tile_step) {
                const int img = tile / per_img, t = tile - img * per_img;
                const int cy = (t / g.tiles_x) * PH * S - f.pad, cx = (t % g.tiles_x) * PW * S - f.pad;
                for (int kb = 0; kb < nkb; kb++) {
                    mbar_wait(&win_empty[wi], wph ^ 1);
                    mbar_expect_tx(&win_full[wi], (uint32_t)T::BYTES);
                    tma_load_4d(win + (size_t)wi * T::BYTES, &tmap_win, &win_full[wi], kb * 64, cx, cy, img);
                    if (++wi == f.ws) { wi = 0; wph ^= 1; }
                    mbar_wait(&b_empty[bi], bph ^ 1);
                    mbar_expect_tx(&b_full[bi], (uint32_t)b_bytes);
                    tma_load_2d(b_st + (size_t)bi * b_bytes, &tmap_b, &b_full[bi], kb * BK, n_blk * g.block_n);
                    if (++bi == f.bs) { bi = 0; bph ^= 1; }
                }
            }
        }
        return;
    }
    // ===== depthwise + MMA + epilogue warps =====
    const int wg = warp >> 2;
    const int by = warp / (PW / 4), bx = warp % (PW / 4);        // 4 x 4 output block of this warp inside the patch
    float acc_mma[NG][32];
#pragma unroll
    for (int gi = 0; gi < NG; gi++)
#pragma unroll
        for (int i = 0; i < 32; i++) acc_mma[gi][i] = 0.f;
    float* stg = stg_s + warp * 16 * STG_LD;
    int wi = 0; uint32_t wph = 0; int bi = 0; uint32_t bph = 0;
    for (int tile = tile0; tile < g.m_blocks; tile += tile_step) {
        const int t = tile % per_img;
        const int oy0 = (t / g.tiles_x) * PH + by * 4, ox0 = (t % g.tiles_x) * PW + bx * 4;
        const bool inside = oy0 < g.Ho && ox0 < g.Wo;            // blocks past the image edge: rows nobody stores
        int b_prev = 0;
        for (int kb = 0; kb < nkb; kb++) {
            const int c0 = kb * 64 + lane * 2;
            const bool cok = c0 < f.C;
            float acc[4][4][2];
#pragma unroll
            for (int i = 0; i < 4; i++)
#pragma unroll
                for (int j = 0; j < 4; j++) { acc[i][j][0] = 0.f; acc[i][j][1] = 0.f; }
            mbar_wait(&win_full[wi], wph);
            if (inside) {
                float wgt[25][2];
                float bias0 = 0.f, bias1 = 0.f;
#pragma unroll
                for (int tp = 0; tp < 25; tp++) {
                    const float2 wv = cok ? *reinterpret_cast<const float2*>(dww_s + (size_t)tp * f.C + c0)
                                          : make_float2(0.f, 0.f);
                    wgt[tp][0] = wv.x; wgt[tp][1] = wv.y;
                }
                if (cok) { const float2 bv = *reinterpret_cast<const float2*>(dww_s + 25 * (size_t)f.C + c0); bias0 = bv.x; bias1 = bv.y; }
                const unsigned char* tile_p = win + (size_t)wi * T::BYTES + lane * 4 +
                                              ((by * 4 * S) * T::IW + bx * 4 * S) * 128;
#pragma unroll
                for (int i = 0; i < 4; i++)
#pragma unroll
                    for (int j = 0; j < 4; j++) { acc[i][j][0] = bias0; acc[i][j][1] = bias1; }
#pragma unroll
                for (int ry = 0; ry < T::WIN_Y; ry++) {
                    float v2[T::WIN_X][2];
#pragma unroll
                    for (int cx = 0; cx < T::WIN_X; cx++) {
                        const uint32_t v = *reinterpret_cast<const uint32_t*>(tile_p + (ry * T::IW + cx) * 128);
                        v2[cx][0] = __uint_as_float(v << 16);
                        v2[cx][1] = __uint_as_float(v & 0xffff0000u);
                    }
#pragma unroll
                    for (int i = 0; i < 4; i++) {
                        const int ky = ry - i * S;                    // compile-time after unrolling
                        if (ky < 0 || ky >= 5) continue;
#pragma unroll
                        for (int kx = 0; kx < 5; kx++) {
#pragma unroll
                            for (int j = 0; j < 4; j++) {
                                acc[i][j][0] = fmaf(v2[j * S + kx][0], wgt[ky * 5 + kx][0], acc[i][j][0]);
                                acc[i][j][1] = fmaf(v2[j * S + kx][1], wgt[ky * 5 + kx][1], acc[i][j][1]);
                            }
                        }
                    }
                }
                if (f.dw_relu) {
#pragma unroll
                    for (int i = 0; i < 4; i++)
#pragma unroll
                        for (int j = 0; j < 4; j++) {
                            acc[i][j][0] = fmaxf(acc[i][j][0], 0.f); acc[i][j][1] = fmaxf(acc[i][j][1], 0.f);
                        }
                }
            }
            // the window slot is free as soon as its values sit in registers
            __syncwarp();
            if (lane == 0) mbar_arrive(&win_empty[wi]);
            if (++wi == f.ws) { wi = 0; wph ^= 1; }
            // the MMAs of the previous K block (they ran under the FMAs above) have read the A stage and their B stage
            if (kb > 0) {
                wgmma_wait<0>();
                if (lane == 0) mbar_arrive(&b_empty[b_prev]);
            }
            // A stage: row = pixel of the patch, 16-byte chunk index XOR (row & 7) (SWIZZLE_128B, K-major).  Rows of
            // blocks past the image edge are zero (their results are never stored).
            {
                unsigned char* a_base = a_st + (lane & 3) * 4;
#pragma unroll
                for (int i = 0; i < 4; i++)
#pragma unroll
                    for (int j = 0; j < 4; j++) {
                        const int row = (by * 4 + i) * PW + bx * 4 + j;
                        *reinterpret_cast<uint32_t*>(a_base + row * 128 + ((((lane >> 2) ^ (row & 7))) << 4)) =
                            pack_bf16(acc[i][j][0], acc[i][j][1]);
                    }
            }
            fence_proxy_async_shared();
            // the four warps of a warpgroup wrote exactly the 64 rows their MMAs read
            asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");
            mbar_wait(&b_full[bi], bph);
#pragma unroll
            for (int gi = 0; gi < NG; gi++) fence_acc(acc_mma[gi]);
            wgmma_fence();
            mma_k_block<NG, LASTW>(acc_mma, smem_u32(a_st) + wg * WG_ROWS * BK * 2, smem_u32(b_st + (size_t)bi * b_bytes),
                                   kb == 0);
            wgmma_commit();
            b_prev = bi;
            if (++bi == f.bs) { bi = 0; bph ^= 1; }
        }
        wgmma_wait<0>();
#pragma unroll
        for (int gi = 0; gi < NG; gi++) fence_acc(acc_mma[gi]);
        if (lane == 0) mbar_arrive(&b_empty[b_prev]);
        warp_epilogue<NG>(g, acc_mma, stg, tile, n_blk, warp * 16, bias_s, nullptr, dest_s);
    }
}

size_t fused_smem_bytes(int ws, int bs, int block_n, int n_pad, int c_dw) {
    return 1024 + (size_t)BM * BK * 2 + (size_t)bs * block_n * BK * 2 + (size_t)ws * DwTile<1, PH, PW, 4, 1>::BYTES +
           (size_t)n_pad * 5 + (size_t)c_dw * 26 * 4 + STG_BYTES + (size_t)(2 * (ws + bs)) * 8 + 64;
}

// ------------------------------------------------------------------ fused 1x1 GEMM -> depthwise 5x5
// InvertedResidualK branch2 head (basenetworks.py:214-218: 1x1, BN, ReLU, dw5x5 stride 2, BN) of the stage-entry
// block whose 1x1 reads the stem output (at most 32 channels) as ONE kernel: the 1x1 output -- the largest activation
// of the network -- never visits HBM.  The 1x1 is recomputed on each item's input window instead: the halo of a
// stride-2 5x5 window re-reads 1.3x the pixels, and 32-channel k16 steps cost the tensor core next to nothing.
// Persistent CTA over (image, tile row, tile column) items of TH x TW output pixels:
//   last warp  TMA producer: the item's window of the 1x1 input, IH x IW pixels x 32 channels (4-D box, zero fill,
//              64-byte swizzle: the K-major wgmma layout of 64-byte rows) into a 2-deep ring
//   the others per 64-channel block of the 1x1 output: the warpgroups multiply 64-pixel row chunks of the window
//              by the block's resident weights (2 x wgmma.m64n64k16, the k16 steps and f32 epilogue of k_gemm_wg:
//              bit-identical to the t_c that k_gemm_wg would write), bias + ReLU, bf16 into the intermediate window
//              (128 bytes per pixel, 16-byte units XOR (pixel & 7)).  Pixels outside the image are written as 0, not
//              relu(bias): the depthwise conv zero-pads ITS input, the 1x1 output.  Then, after a barrier, the
//              depthwise FMA loop of k_dwconv5_tma (dw5_block, one 4 x BW output block per warp) on that block; a
//              second barrier before the next block's epilogue overwrites the intermediate.
// Resident per CTA, staged before the grid-dependency wait: the 1x1 weights [cblks * 64][32] bf16 (64-byte swizzle)
// and bias, the depthwise weights [25][C] f32 and bias.
template <int S, int TH, int TW, int BW>
struct PwDwTile {
    static constexpr int IH = (TH - 1) * S + 5, IW = (TW - 1) * S + 5;
    static constexpr int NPIX = IH * IW;
    static constexpr int CHUNKS = (NPIX + WG_ROWS - 1) / WG_ROWS;      // 64-row wgmma chunks of the window
    static constexpr int IN_BYTES = CHUNKS * WG_ROWS * 64;             // 64-byte rows; the tail rows are never stored
    static constexpr int MID_BYTES = NPIX * 128;
    static constexpr int NSTAGE = 2;
    static constexpr int WARPS = (TH / 4) * (TW / BW);               // consumer warps: one 4 x BW depthwise block each
    static constexpr int WGS = WARPS / 4;                             // ... forming this many wgmma warpgroups
    static constexpr int THREADS = 32 * (WARPS + 1);
    static_assert(WARPS % 4 == 0, "whole warpgroups");
};
constexpr int PWDW_K = 32;       // 1x1 input channels the window carries (64-byte pixel rows)

struct PwDwArgs {
    DwArgs dw;                   // the depthwise op (dw.in: the elided 1x1 output, not read)
    const __nv_bfloat16* w1; int ldw1, n1;   // 1x1 weights [n1][ldw1] bf16 (ldw1 <= PWDW_K), bias [n1] f32
    const float* b1; int relu1;
    int Hin, Win;                // the 1x1 input == the depthwise input grid
    int cblks;                   // 64-channel blocks of the depthwise
};

// K-major, SWIZZLE_64B shared-memory matrix descriptor of wgmma: 64-byte rows, SBO = 512 B (8 rows), layout 64B (2)
__device__ __forceinline__ uint64_t make_smem_desc_64b(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= static_cast<uint64_t>((smem_addr >> 4) & 0x3fffu);
    d |= static_cast<uint64_t>(1u) << 16;
    d |= static_cast<uint64_t>(512u >> 4) << 32;
    d |= static_cast<uint64_t>(2u) << 62;
    return d;
}

size_t pw_dw_smem_bytes(int in_bytes, int mid_bytes, int cblks, int c_dw) {
    return 1024 + 2 * (size_t)in_bytes + (size_t)mid_bytes + (size_t)cblks * 64 * (PWDW_K * 2 + 4) + (size_t)c_dw * 26 * 4;
}

template <int S, int TH, int TW, int BW>
__global__ void __launch_bounds__(PwDwTile<S, TH, TW, BW>::THREADS, 1)
k_pw_dw(const __grid_constant__ CUtensorMap tmap_in, PwDwArgs f) {
    using T = PwDwTile<S, TH, TW, BW>;
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    // align with pointer arithmetic on the array itself: the compiler keeps the shared address space (LDS / STS
    // instead of generic loads and stores)
    unsigned char* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    __shared__ uint64_t full[T::NSTAGE], empty[T::NSTAGE];
    const DwArgs& a = f.dw;
    const int C = a.C8 * 8;
    const int c_pad = f.cblks * 64;
    // the wgmma operands (window ring, 1x1 weights) start on multiples of 4 KB, as the swizzle patterns require
    unsigned char* in_s = smem;                                       // [NSTAGE][IN_BYTES]
    unsigned char* w1_s = in_s + T::NSTAGE * T::IN_BYTES;             // [c_pad][64 B]
    unsigned char* mid = w1_s + (size_t)c_pad * PWDW_K * 2;           // [NPIX][128 B]
    float* b1_s = reinterpret_cast<float*>(mid + T::MID_BYTES);       // [c_pad]
    float* dww_s = b1_s + c_pad;                                      // [25][C] + bias [C]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (warp == T::WARPS && lane == 0) tma_prefetch_desc(&tmap_in);
    // 1x1 weights: row n, 16-byte unit u at u ^ ((n >> 1) & 3) (the 64-byte swizzle TMA would have produced)
    for (int i = threadIdx.x; i < c_pad * (PWDW_K / 8); i += T::THREADS) {
        const int n = i / (PWDW_K / 8), u = i % (PWDW_K / 8);
        uint4 v = make_uint4(0u, 0u, 0u, 0u);
        if (n < f.n1 && u * 8 < f.ldw1) v = *reinterpret_cast<const uint4*>(f.w1 + (size_t)n * f.ldw1 + u * 8);
        *reinterpret_cast<uint4*>(w1_s + n * 64 + ((u ^ ((n >> 1) & 3)) << 4)) = v;
    }
    for (int i = threadIdx.x; i < c_pad; i += T::THREADS) b1_s[i] = i < f.n1 ? f.b1[i] : 0.f;
    for (int i = threadIdx.x; i < 25 * C; i += T::THREADS) dww_s[i] = a.weight[i];
    for (int i = threadIdx.x; i < C; i += T::THREADS) dww_s[25 * C + i] = a.bias[i];
    if (threadIdx.x == 0) {
        for (int s = 0; s < T::NSTAGE; s++) { mbar_init(&full[s], 1); mbar_init(&empty[s], T::WARPS); }
        fence_barrier_init();
    }
    fence_proxy_async_shared();          // the weight tile is read by wgmma (async proxy)
    __syncthreads();
    pdl_launch_dependents();
    pdl_wait();

    const int tiles_x = (a.Wout + TW - 1) / TW, tiles_y = (a.Hout + TH - 1) / TH;
    const int per_img = tiles_y * tiles_x;
    const int total = a.B * per_img;

    if (warp == T::WARPS) {
        // ===== TMA producer =====
        if (lane == 0) {
            int s = 0; uint32_t ph = 0;
            for (int w = blockIdx.x; w < total; w += gridDim.x) {
                const int b = w / per_img, t = w - b * per_img;
                const int ty = t / tiles_x, tx = t - ty * tiles_x;
                mbar_wait(&empty[s], ph ^ 1);
                mbar_expect_tx(&full[s], (uint32_t)(T::NPIX * PWDW_K * 2));
                tma_load_4d(in_s + (size_t)s * T::IN_BYTES, &tmap_in, &full[s], 0, tx * TW * S - a.pad,
                            ty * TH * S - a.pad, b);
                if (++s == T::NSTAGE) { s = 0; ph ^= 1; }
            }
        }
        return;
    }
    // ===== consumer warps: 1x1 row chunks (per warpgroup), then one 4 x BW depthwise block each =====
    const int wg = warp >> 2;
    const int by = warp / (TW / BW), bx = warp % (TW / BW);
    const int q = lane & 3;
    float acc[32];
#pragma unroll
    for (int i = 0; i < 32; i++) acc[i] = 0.f;
    int s = 0; uint32_t ph = 0;
    for (int w = blockIdx.x; w < total; w += gridDim.x) {
        const int b = w / per_img, t = w - b * per_img;
        const int ty = t / tiles_x, tx = t - ty * tiles_x;
        const int iy0 = ty * TH * S - a.pad, ix0 = tx * TW * S - a.pad;
        const uint32_t a_s = smem_u32(in_s + (size_t)s * T::IN_BYTES);
        mbar_wait(&full[s], ph);
        for (int cb = 0; cb < f.cblks; cb++) {
            const uint32_t b_s = smem_u32(w1_s + (size_t)cb * 64 * PWDW_K * 2);
            for (int mc = wg; mc < T::CHUNKS; mc += T::WGS) {
                fence_acc(acc);
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < PWDW_K / MMA_K; k++)
                    wgmma_n64(acc, make_smem_desc_64b(a_s + mc * WG_ROWS * PWDW_K * 2 + k * MMA_K * 2),
                              make_smem_desc_64b(b_s + k * MMA_K * 2), k == 0 ? 0u : 1u);
                wgmma_commit();
                wgmma_wait<0>();
                fence_acc(acc);
                // epilogue (k_gemm_wg's): bias + ReLU in f32, bf16; rows r and r + 8 of this warp's 16
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    const int r = mc * WG_ROWS + (warp & 3) * 16 + (lane >> 2) + 8 * h;
                    if (r >= T::NPIX) continue;
                    const int wy = r / T::IW, wx = r - wy * T::IW;
                    const bool inside = (unsigned)(iy0 + wy) < (unsigned)f.Hin && (unsigned)(ix0 + wx) < (unsigned)f.Win;
                    unsigned char* row = mid + r * 128 + q * 4;
#pragma unroll
                    for (int j = 0; j < 8; j++) {
                        const float2 bb = *reinterpret_cast<const float2*>(b1_s + cb * 64 + 8 * j + 2 * q);
                        float v0 = acc[4 * j + 2 * h] + bb.x, v1 = acc[4 * j + 2 * h + 1] + bb.y;
                        if (f.relu1) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
                        *reinterpret_cast<uint32_t*>(row + ((j ^ (r & 7)) << 4)) = inside ? pack_bf16(v0, v1) : 0u;
                    }
                }
            }
            // the window slot is free once the last block's MMAs have read it
            if (cb == f.cblks - 1) {
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty[s]);
            }
            asm volatile("bar.sync 1, %0;" ::"n"(32 * T::WARPS) : "memory");
            const int c0 = cb * 64 + lane * 2;
            const int oy0 = ty * TH + by * 4, ox0 = tx * TW + bx * BW;
            if (oy0 < a.Hout && ox0 < a.Wout && c0 < C) {
                float wgt[25][2];
#pragma unroll
                for (int tp = 0; tp < 25; tp++) {
                    const float2 wv = *reinterpret_cast<const float2*>(dww_s + (size_t)tp * C + c0);
                    wgt[tp][0] = wv.x; wgt[tp][1] = wv.y;
                }
                const float2 bv = *reinterpret_cast<const float2*>(dww_s + 25 * (size_t)C + c0);
                dw5_block<S, BW, T::IW, true>(a, mid, (by * 4 * S) * T::IW + bx * BW * S, lane, wgt, bv.x, bv.y,
                                              b, oy0, ox0, c0);
            }
            // every depthwise read of the intermediate is done before the next block's epilogue overwrites it
            asm volatile("bar.sync 1, %0;" ::"n"(32 * T::WARPS) : "memory");
        }
        if (++s == T::NSTAGE) { s = 0; ph ^= 1; }
    }
}

// stride 2, 8 x 16 output tiles (DwS2's shape: the smaller halo): 2 x 45 KB window ring + 85 KB intermediate + the
// resident weights -> 1 CTA per SM.  4 x 2 depthwise blocks: 16 consumer warps (four warpgroups) instead of the 8
// of 4 x 4 blocks -- both phases are latency bound at one CTA per SM, twice the warps hide twice the latency
constexpr int PWDW_TH = 8, PWDW_TW = 16, PWDW_BW = 2;
using PwDwS2 = PwDwTile<2, PWDW_TH, PWDW_TW, PWDW_BW>;

// every (column groups, last group width) instantiation, indexed [NG - 1][LASTW / 16 - 1]: any block_n that is a
// multiple of 16 up to 256 (192 for the fused op)
using GemmKernel = decltype(&k_gemm_wg<1, 16>);
const GemmKernel GEMM_KERNELS[4][4] = {
    {k_gemm_wg<1, 16>, k_gemm_wg<1, 32>, k_gemm_wg<1, 48>, k_gemm_wg<1, 64>},
    {k_gemm_wg<2, 16>, k_gemm_wg<2, 32>, k_gemm_wg<2, 48>, k_gemm_wg<2, 64>},
    {k_gemm_wg<3, 16>, k_gemm_wg<3, 32>, k_gemm_wg<3, 48>, k_gemm_wg<3, 64>},
    {k_gemm_wg<4, 16>, k_gemm_wg<4, 32>, k_gemm_wg<4, 48>, k_gemm_wg<4, 64>}};
using DwGemmKernel = decltype(&k_dw_gemm<1, 1, 16>);
const DwGemmKernel DW_GEMM_KERNELS[3][4] = {
    {k_dw_gemm<1, 1, 16>, k_dw_gemm<1, 1, 32>, k_dw_gemm<1, 1, 48>, k_dw_gemm<1, 1, 64>},
    {k_dw_gemm<1, 2, 16>, k_dw_gemm<1, 2, 32>, k_dw_gemm<1, 2, 48>, k_dw_gemm<1, 2, 64>},
    {k_dw_gemm<1, 3, 16>, k_dw_gemm<1, 3, 32>, k_dw_gemm<1, 3, 48>, k_dw_gemm<1, 3, 64>}};
// block_n (a multiple of 16) -> {NG - 1, LASTW / 16 - 1}
inline int tile_groups(int block_n) { return (block_n + NGROUP - 1) / NGROUP - 1; }
inline int tile_last(int block_n) { return (block_n - tile_groups(block_n) * NGROUP) / 16 - 1; }

// ------------------------------------------------------------------ input conv: f32 NCHW [B,3,H,W] -> bf16 NHWC
struct InConvArgs {
    const float* in; __nv_bfloat16* out; int ld_out;
    // raw-image variant: uint8 [B][H][W][3] (what PIL / the decoder of a video stream delivers); the kernel applies
    // torchvision's ToTensor + Normalize (transforms/__init__.py:26-33) on load: ((u / 255) - mean[c]) / std[c]
    const uint8_t* in_u8; float mean[3], stdev[3];
    const float* weight;   // [3*k*k][C8*8] (tap-major)
    const float* bias;     // [C8*8]
    int B, Hin, Win, Hout, Wout, C8, kernel, stride, pad, relu;
};

template <int KS, bool U8>
__global__ void __launch_bounds__(256) k_input_conv(InConvArgs a) {
    // one thread = one output pixel, all output channels: the 3*k*k input samples are loaded once (registers for
    // k = 3, thread-local memory for k = 7) and reused for every 8-channel group; weights are broadcast reads
    // from shared memory
    extern __shared__ __align__(16) float s_w[];      // [3*k*k][C] weights + [C] bias
    constexpr int TAPS = 3 * KS * KS;
    const int C = a.C8 * 8;
    const int n_w = TAPS * C;
    for (int i = threadIdx.x; i < n_w; i += blockDim.x) s_w[i] = a.weight[i];
    for (int i = threadIdx.x; i < C; i += blockDim.x) s_w[n_w + i] = a.bias[i];
    // raw images: the 256 possible values of a channel, normalised once per CTA with IEEE division / subtraction
    // (bit-identical to torchvision's ToTensor + Normalize on the host) -> one byte load + one table read per sample
    float* s_lut = s_w + n_w + C;                     // [3][256]
    if (U8)
        for (int i = threadIdx.x; i < 256; i += blockDim.x) {
            const float x = __fdiv_rn((float)i, 255.f);
#pragma unroll
            for (int c = 0; c < 3; c++) s_lut[c * 256 + i] = __fdiv_rn(__fsub_rn(x, a.mean[c]), a.stdev[c]);
        }
    pdl_launch_dependents();
    pdl_wait();
    __syncthreads();
    const long long total = (long long)a.B * a.Hout * a.Wout;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total;
         t += (long long)gridDim.x * blockDim.x) {
        long long p = t;
        const int ox = (int)(p % a.Wout); p /= a.Wout;
        const int oy = (int)(p % a.Hout);
        const int b = (int)(p / a.Hout);
        float in[TAPS];
        if (U8) {
            // HWC bytes: the three channels of a pixel are adjacent; one row pointer per ky, one pixel pointer per kx
#pragma unroll
            for (int ky = 0; ky < KS; ky++) {
                const int iy = oy * a.stride - a.pad + ky;
                const bool oky = iy >= 0 && iy < a.Hin;
                const uint8_t* rowp = a.in_u8 + ((size_t)b * a.Hin + (oky ? iy : 0)) * a.Win * 3;
#pragma unroll
                for (int kx = 0; kx < KS; kx++) {
                    const int ix = ox * a.stride - a.pad + kx;
                    const bool ok = oky && ix >= 0 && ix < a.Win;
                    const uint8_t* px = rowp + (ok ? ix : 0) * 3;
#pragma unroll
                    for (int ci = 0; ci < 3; ci++)
                        in[(ci * KS + ky) * KS + kx] = ok ? s_lut[ci * 256 + __ldg(px + ci)] : 0.f;
                }
            }
        } else {
#pragma unroll
            for (int ci = 0; ci < 3; ci++) {
                const float* plane = a.in + ((size_t)b * 3 + ci) * a.Hin * a.Win;
#pragma unroll
                for (int ky = 0; ky < KS; ky++) {
                    const int iy = oy * a.stride - a.pad + ky;
#pragma unroll
                    for (int kx = 0; kx < KS; kx++) {
                        const int ix = ox * a.stride - a.pad + kx;
                        const bool ok = iy >= 0 && iy < a.Hin && ix >= 0 && ix < a.Win;
                        in[(ci * KS + ky) * KS + kx] = ok ? __ldg(plane + (size_t)iy * a.Win + ix) : 0.f;
                    }
                }
            }
        }
        __nv_bfloat16* orow = a.out + ((size_t)(b * a.Hout + oy) * a.Wout + ox) * a.ld_out;
        for (int c8 = 0; c8 < a.C8; c8++) {
            float acc[8];
            const float4 b0 = *reinterpret_cast<const float4*>(s_w + n_w + c8 * 8);
            const float4 b1 = *reinterpret_cast<const float4*>(s_w + n_w + c8 * 8 + 4);
            acc[0] = b0.x; acc[1] = b0.y; acc[2] = b0.z; acc[3] = b0.w;
            acc[4] = b1.x; acc[5] = b1.y; acc[6] = b1.z; acc[7] = b1.w;
#pragma unroll
            for (int tp = 0; tp < TAPS; tp++) {
                const float4 w0 = *reinterpret_cast<const float4*>(s_w + (size_t)tp * C + c8 * 8);
                const float4 w1 = *reinterpret_cast<const float4*>(s_w + (size_t)tp * C + c8 * 8 + 4);
                const float v = in[tp];
                acc[0] = fmaf(v, w0.x, acc[0]); acc[1] = fmaf(v, w0.y, acc[1]);
                acc[2] = fmaf(v, w0.z, acc[2]); acc[3] = fmaf(v, w0.w, acc[3]);
                acc[4] = fmaf(v, w1.x, acc[4]); acc[5] = fmaf(v, w1.y, acc[5]);
                acc[6] = fmaf(v, w1.z, acc[6]); acc[7] = fmaf(v, w1.w, acc[7]);
            }
#pragma unroll
            for (int j = 0; j < 8; j++) acc[j] = act_f(acc[j], a.relu);
            uint4 o;
            o.x = pack_bf16(acc[0], acc[1]); o.y = pack_bf16(acc[2], acc[3]);
            o.z = pack_bf16(acc[4], acc[5]); o.w = pack_bf16(acc[6], acc[7]);
            *reinterpret_cast<uint4*>(orow + c8 * 8) = o;
        }
    }
}

// dynamic shared memory of k_input_conv: weights [3*k*k][C] + bias [C] + the u8 normalisation table [3][256]
constexpr int INCONV_SMEM_MAX = 226 * 1024;
inline size_t input_conv_smem_bytes(int kernel, int c8) {
    return sizeof(float) * ((size_t)3 * kernel * kernel * c8 * 8 + (size_t)c8 * 8 + 3 * 256);
}

__global__ void k_f32_to_bf16(const float* in, __nv_bfloat16* out, long long n) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        out[i] = __float2bfloat16_rn(in[i]);
}

__global__ void k_bf16_to_f32(const __nv_bfloat16* in, float* out, long long n) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        out[i] = __bfloat162float(in[i]);
}

// ------------------------------------------------------------------ host side
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// bf16 tensor map of `rank` dimensions (innermost first; row pitches in elements); a failure names the map and its shape
int encode_tmap(CUtensorMap* map, const char* what, const void* base, int rank, const cuuint64_t* dims,
                const cuuint64_t* ld, const cuuint32_t* box, const cuuint32_t* estr, CUtensorMapSwizzle swz,
                CUtensorMapL2promotion l2) {
    static PFN_encodeTiled fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<PFN_encodeTiled>(p);
    }
    if (!fn) { pifpaf::set_error("cuTensorMapEncodeTiled entry point not available"); return PIFPAF_E_CUDA; }
    cuuint64_t strides[3];
    for (int i = 0; i + 1 < rank; i++) strides[i] = ld[i] * 2;
    const CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, rank, const_cast<void*>(base), dims, strides, box, estr,
                          CU_TENSOR_MAP_INTERLEAVE_NONE, swz, l2, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        char shape[256] = "";      // " dim/box" per dimension, then " ld" per pitch: at most 4 x 32 + 3 x 22 bytes
        for (int i = 0; i < rank; i++)
            snprintf(shape + strlen(shape), sizeof(shape) - strlen(shape), " %llu/%u", (unsigned long long)dims[i], box[i]);
        for (int i = 0; i + 1 < rank; i++)
            snprintf(shape + strlen(shape), sizeof(shape) - strlen(shape), " ld=%llu", (unsigned long long)ld[i]);
        pifpaf::set_error("cuTensorMapEncodeTiled (%s) failed (%d): dim/box%s base=%p", what, (int)r, shape, base);
        return PIFPAF_E_CUDA;
    }
    return PIFPAF_OK;
}

// 2-D bf16 row-major view [rows][cols] with row pitch ld (elements); box = [box_rows][64 cols], 128B swizzle
int make_tmap(CUtensorMap* map, const void* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows) {
    const cuuint64_t dims[2] = {cols, rows};
    const cuuint32_t box[2] = {BK, box_rows}, estr[2] = {1, 1};
    return encode_tmap(map, "gemm", base, 2, dims, &ld, box, estr, CU_TENSOR_MAP_SWIZZLE_128B,
                       CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
}

// 2-D bf16 row-major view, un-swizzled box [box_rows][box_cols] (dense rows in shared memory)
int make_tmap_plain(CUtensorMap* map, const void* base, uint64_t rows, uint64_t cols, uint64_t ld,
                    uint32_t box_cols, uint32_t box_rows) {
    const cuuint64_t dims[2] = {cols, rows};
    const cuuint32_t box[2] = {box_cols, box_rows}, estr[2] = {1, 1};
    return encode_tmap(map, "plain", base, 2, dims, &ld, box, estr, CU_TENSOR_MAP_SWIZZLE_NONE,
                       CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
}

// 2-D bf16 output view for the TMA-store epilogue: box = 16 rows x 16 columns (32 bytes), 32-byte swizzle
int make_tmap_store(CUtensorMap* map, const void* base, uint64_t rows, uint64_t cols, uint64_t ld) {
    const cuuint64_t dims[2] = {cols, rows};
    const cuuint32_t box[2] = {OUT_BOX_COLS, OUT_BOX_ROWS}, estr[2] = {1, 1};
    return encode_tmap(map, "store", base, 2, dims, &ld, box, estr, CU_TENSOR_MAP_SWIZZLE_32B,
                       CU_TENSOR_MAP_L2_PROMOTION_NONE);
}

// 4-D bf16 NHWC activation view {C, W, H, B} for implicit-GEMM convolutions: box = 64 channels x the
// input window of a PH x PW output patch, traversed with the conv stride
int make_tmap_conv(CUtensorMap* map, const void* base, uint64_t c, uint64_t w, uint64_t h, uint64_t b, uint64_t ld,
                   int stride) {
    const cuuint64_t dims[4] = {c, w, h, b}, lds[3] = {ld, w * ld, h * w * ld};
    const cuuint32_t box[4] = {BK, (cuuint32_t)((PW - 1) * stride + 1), (cuuint32_t)((PH - 1) * stride + 1), 1};
    const cuuint32_t estr[4] = {1, (cuuint32_t)stride, (cuuint32_t)stride, 1};
    return encode_tmap(map, "conv", base, 4, dims, lds, box, estr, CU_TENSOR_MAP_SWIZZLE_128B,
                       CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
}

// 4-D bf16 NHWC view {C, W, H, B}, dense (un-swizzled) box of 64 channels x box_w x box_h pixels.
// No L2 promotion: the 128-byte channel block of a pixel is all the kernel wants from that pixel for a long time
// (the channel block is the slowest work index) and pixel strides of 352 / 704 bytes leave most blocks straddling
// 128-byte lines: a wider promotion fetches bytes nobody reads.
// box_c / swz: k_pw_dw's window of a 32-channel 1x1 input is a 64-byte swizzled box of 32 channels (its wgmma layout)
int make_tmap_dw(CUtensorMap* map, const void* base, uint64_t c, uint64_t w, uint64_t h, uint64_t b, uint64_t ld,
                 uint32_t box_w, uint32_t box_h, uint32_t box_c = 64,
                 CUtensorMapSwizzle swz = CU_TENSOR_MAP_SWIZZLE_NONE) {
    const cuuint64_t dims[4] = {c, w, h, b}, lds[3] = {ld, w * ld, h * w * ld};
    const cuuint32_t box[4] = {box_c, box_w, box_h, 1}, estr[4] = {1, 1, 1, 1};
    return encode_tmap(map, "dw", base, 4, dims, lds, box, estr, swz, CU_TENSOR_MAP_L2_PROMOTION_NONE);
}

// every kernel launch of net.cu: with (or without) the programmatic-stream-serialization attribute, counted and checked
template <typename... KArgs, typename... Args>
int launch_k(bool pdl, void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    int n = 0;
    if (pdl) {
        attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[n].val.programmaticStreamSerializationAllowed = 1;
        n++;
    }
    cfg.attrs = attr; cfg.numAttrs = n;
    PIFPAF_CUDA_TRY(cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...));
    PIFPAF_LAUNCH_CHECK();
    return PIFPAF_OK;
}

// the TMA depthwise kernels, one entry per instantiation: choose_dw_kernels picks the entry of an op (pifpaf_net_dwconv
// encodes its box), the launch takes kernel, block and grid from it, pifpaf_net_create sets its shared-memory limit
using DwTmaKernel = decltype(&k_dwconv5_tma<1, DW1_TH, DW1_TW, 4, 3>);
struct DwTmaVariant {
    DwTmaKernel kernel;
    int threads;
    int smem;                 // dynamic shared memory (DW_K5_S2_CBF: the limit; a launch takes what its weights need)
    int th, tw;               // output tile
    int ctas_per_sm;          // persistent grid == resident CTAs (by shared memory)
    uint32_t box_w, box_h;    // input window (TMA box)
};
enum { DW_K5_S1, DW_K5_S2, DW_K5_S2_CBF, DW_K3_S1, DW_K3_S2, DW_K5_S1_D2, DW_TMA_VARIANTS };
const DwTmaVariant DW_TMA[DW_TMA_VARIANTS] = {
    {k_dwconv5_tma<1, DW1_TH, DW1_TW, 4, 3>, DwS1::THREADS, DwS1::SMEM, DW1_TH, DW1_TW, 2, DwS1::IW, DwS1::IH},
    {k_dwconv5_tma<2, DW2_TH, DW2_TW, 4, 2>, DwS2::THREADS, DwS2::SMEM, DW2_TH, DW2_TW, 1, DwS2::IW, DwS2::IH},
    // channel-block-fastest item order with the weights staged in shared memory (PIFPAF_DW_CBF=1): DW_K5_S2's
    // window and grid, chosen at emit while the weights fit
    {k_dwconv5_tma<2, DW2_TH, DW2_TW, 4, 2, true>, DwS2::THREADS, 226 * 1024, DW2_TH, DW2_TW, 1, DwS2::IW, DwS2::IH},
    {k_dwconv5_tma<1, DW1_TH, DW1_TW, 4, 4, false, 3>, DwS1K3::THREADS, DwS1K3::SMEM, DW1_TH, DW1_TW, 2, DwS1K3::IW,
     DwS1K3::IH},
    {k_dwconv5_tma<2, DW2_TH, DW2_TW, 4, 3, false, 3>, DwS2K3::THREADS, DwS2K3::SMEM, DW2_TH, DW2_TW, 1, DwS2K3::IW,
     DwS2K3::IH},
    {k_dwconv5_tma<1, DW1_TH, DW1_TW, 4, 2, false, 5, 2>, DwS1D2::THREADS, DwS1D2::SMEM, DW1_TH, DW1_TW, 2, DwS1D2::IW,
     DwS1D2::IH}};

// the stem instantiations, indexed [U8][KS / 2] (KS = 1, 3, 5, 7)
using InConvKernel = decltype(&k_input_conv<1, false>);
const InConvKernel INPUT_CONV_KERNELS[2][4] = {
    {k_input_conv<1, false>, k_input_conv<3, false>, k_input_conv<5, false>, k_input_conv<7, false>},
    {k_input_conv<1, true>, k_input_conv<3, true>, k_input_conv<5, true>, k_input_conv<7, true>}};

struct Tensor { int h, w, c; __nv_bfloat16* data; };

// the values are the op kinds pifpaf_net_forward_timed reports (a fused 1x1 -> depthwise pair: OP_FUSED)
enum OpKind { OP_INPUT_CONV, OP_GEMM, OP_DW, OP_FUSED, OP_MAXPOOL };

struct Op {
    OpKind kind;
    // gemm
    GemmArgs g{};
    CUtensorMap tmap_a{}, tmap_b{}, tmap_src{};
    int a_tensor = -1; int rows_per_image = 0; int tiles_per_image = 0;
    size_t smem = 0;                 // dynamic shared memory: k_gemm_wg, k_dw_gemm, the TMA depthwise kernel (dw_tma)
    // TMA-store epilogue (g.tma_store): the output views {base, columns, row pitch}, one per store map; the maps
    // bound rows at batch * rows_per_image and are re-encoded when the batch changes (store_rows: the M they hold)
    struct StoreView { const __nv_bfloat16* base; int cols; int ld; };
    std::vector<StoreView> store_views;
    StoreMaps smaps{};
    int store_rows = -1;
    // dw, max pool
    DwArgs dw{};
    CUtensorMap tmap_dw{};
    const DwTmaVariant* dw_tma = nullptr;     // TMA route of a depthwise op (choose_dw_kernels; nullptr: none)
    void (*dw_simt5)(DwArgs) = nullptr;       // its SIMT route: k_dwconv5<S> (nullptr: k_dwconv)
    int dw_dil = 1;                           // depthwise tap spacing (> 1: DW_K5_S1_D2 or k_dwconv)
    // fused depthwise -> GEMM (OP_FUSED): g + tmap_dw (windows) + tmap_b
    FusedArgs fu{};
    // input conv
    InConvArgs ic{};
    double flops_per_image = 0;
    double bytes_per_image = 0;      // algorithmic activation bytes (inputs once + outputs once)
    double weight_bytes = 0;
    int n_real = 0;                  // output channels that are not padding (emit_gemm)
    double a_bytes_per_image = 0;    // GEMM: the input part of bytes_per_image
    double dw_out_bytes_per_image = 0;   // depthwise: the output part of bytes_per_image
    std::vector<int> touches;        // tensor ids the op reads or writes (-1: none)
    // fused 1x1 -> depthwise (plan_pw_dw): the GEMM op is elided (not launched) and the depthwise op right after it
    // launches k_pw_dw with pw + tmap_pw instead
    bool elided = false;
    bool pw_dw = false;
    PwDwArgs pw{};
    CUtensorMap tmap_pw{};
    size_t pw_smem = 0;
    double pw_flops_per_image = 0, pw_bytes_per_image = 0, pw_weight_bytes = 0;
};

}  // namespace

struct pifpaf_net {
    int device = 0, max_batch = 0, n_sm = 132;
    std::vector<Tensor> tensors;
    std::vector<Op> ops;
    std::vector<void*> owned;            // device allocations (weights, biases, tables)
    // heads
    int n_heads = 0;
    // head outputs, optionally double buffered: forward i writes head_out[i & 1] so that a decode of forward i-1
    // (another stream) may still read the other set (pifpaf_net_set_head_buffers)
    float* head_out[2][4] = {{nullptr, nullptr, nullptr, nullptr}, {nullptr, nullptr, nullptr, nullptr}};
    int head_buffers = 1, head_cur = 0;
    size_t head_elems[4] = {0, 0, 0, 0};
    bool setup_synced = false;           // build-time memsets / uploads (legacy stream) ordered before the first forward
    int sm_limit = 0;                    // > 0: persistent grids use at most this many SMs
    bool pdl = true;                     // programmatic dependent launch between the ops of a forward (PIFPAF_PDL=0: off)
    int gemm_res_stages = 0;             // weights-resident GEMMs: split N further until this many A stages fit (PIFPAF_GEMM_RES_STAGES)
    bool dw_cbf = false;                 // stride-2 depthwise: channel-block-fastest item order (PIFPAF_DW_CBF=1)
    bool gemm_tma_store = true;          // plain / scatter 1x1 GEMMs store through TMA (PIFPAF_GEMM_TMA_STORE=0: per-lane stores)
    bool fuse_pw_dw = true;              // 1x1 -> stride-2 depthwise pairs run as k_pw_dw (PIFPAF_FUSE_PW_DW=0: two kernels)
    size_t pw_dw_planned = 0;            // ops.size() when plan_pw_dw last ran
    int elided_batch = 0;                // > 0: the last forward elided GEMMs (at this batch); pifpaf_net_tap_tensor re-runs them
    int head_fields[4] = {0, 0, 0, 0}, head_comp[4] = {0, 0, 0, 0}, head_h = 0, head_w = 0;
    int in_h = 0, in_w = 0;
};

namespace {

template <typename T>
int net_alloc(pifpaf_net* net, T** p, size_t n, bool zero) {
    PIFPAF_TRY(pifpaf::dev_alloc(p, n, net->owned));
    net->setup_synced = false;
    if (zero) {
        const cudaError_t e = cudaMemset(*p, 0, sizeof(T) * (n ? n : 1));
        if (e != cudaSuccess) { pifpaf::set_error("cudaMemset failed: %s", cudaGetErrorString(e)); return PIFPAF_E_CUDA; }
    }
    return PIFPAF_OK;
}

template <typename T>
int net_upload(pifpaf_net* net, T** p, const std::vector<T>& host) {
    int rc = net_alloc(net, p, host.size(), false);
    if (rc != PIFPAF_OK) return rc;
    cudaError_t e = cudaMemcpy(*p, host.data(), sizeof(T) * host.size(), cudaMemcpyHostToDevice);
    if (e != cudaSuccess) { pifpaf::set_error("cudaMemcpy failed: %s", cudaGetErrorString(e)); return PIFPAF_E_CUDA; }
    return PIFPAF_OK;
}

inline int pad8(int v) { return (v + 7) & ~7; }
inline int pad16(int v) { return (v + 15) & ~15; }

// choose the GEMM N tile (<= 256, multiple of 16): the LARGEST tile whose padded work is within
// 10 % of the minimum over all tilings (tiny tiles waste the epilogue and the weight-resident mode; N = 368 must
// become 2 x 192, not 23 x 16)
void choose_block_n(int n_out, int* block_n, int* n_blocks) {
    const int np = pad16(n_out);
    long min_cost = -1;
    for (int nb = 1; nb <= np / 16; nb++) {
        const int bn = pad16((np + nb - 1) / nb);
        if (bn > 256) continue;
        const long cost = (long)bn * nb;
        if (min_cost < 0 || cost < min_cost) min_cost = cost;
    }
    for (int nb = 1; nb <= np / 16; nb++) {
        const int bn = pad16((np + nb - 1) / nb);
        if (bn > 256) continue;
        if ((long)bn * nb * 100 <= min_cost * 110) { *block_n = bn; *n_blocks = nb; return; }
    }
    *block_n = 16; *n_blocks = np / 16;
}

constexpr size_t GEMM_SMEM_BUDGET = 222 * 1024;

// STG_BYTES: the f32 staging tiles of the per-lane epilogue, or the bf16 output chunks of the TMA-store epilogue, which
// fit in the same bytes -- both epilogues get the same ring depth and weight residency
size_t gemm_smem_bytes(int block_n, int n_blocks, int stages, bool shuffle, bool b_resident = false, int num_k_blocks = 0) {
    const size_t b_stage = b_resident ? 0 : (size_t)block_n * BK * 2;
    const size_t b_res = b_resident ? (size_t)num_k_blocks * block_n * BK * 2 : 0;
    return 1024 + (size_t)stages * (BM * BK * 2 + b_stage) + b_res + (shuffle ? 2 * (size_t)BM * block_n * 2 : 0) +
           (size_t)n_blocks * block_n * 5 + STG_BYTES + (2 * stages + 5) * 8 + 64;      // bias (4 B) + scatter table (1 B) per column
}

int choose_stages(int block_n, int n_blocks, int num_k_blocks, bool shuffle) {
    int stages = std::min(8, std::max(2, num_k_blocks * 2));
    while (stages > 2 && gemm_smem_bytes(block_n, n_blocks, stages, shuffle) > GEMM_SMEM_BUDGET) stages--;
    return stages;
}

// A stages of the weights-resident mode: as many as fit next to the whole weight tile (at most 8); 0 if 3 do not
int resident_stages(int block_n, int n_blocks, int num_k_blocks, bool shuffle) {
    if (gemm_smem_bytes(block_n, n_blocks, 3, shuffle, true, num_k_blocks) > GEMM_SMEM_BUDGET) return 0;
    int stages = 8;
    while (gemm_smem_bytes(block_n, n_blocks, stages, shuffle, true, num_k_blocks) > GEMM_SMEM_BUDGET) stages--;
    return stages;
}

// ring depth and shared memory of a GEMM op, once its mode is set: weights-resident mode if the whole weight tile plus
// >= 3 A stages (and the pass-through double buffer) fit; implicit convolutions and the heads stream their weights
void plan_gemm_smem(Op& op) {
    GemmArgs& g = op.g;
    const bool src_tma = g.src_tma != 0;
    const int res = g.conv_k == 0 && g.mode != MODE_HEADS ? resident_stages(g.block_n, g.n_blocks, g.num_k_blocks, src_tma) : 0;
    g.b_resident = res > 0 ? 1 : 0;
    g.stages = res > 0 ? res : choose_stages(g.block_n, g.n_blocks, g.num_k_blocks, src_tma);
    op.smem = gemm_smem_bytes(g.block_n, g.n_blocks, g.stages, src_tma, res > 0, g.num_k_blocks);
}

// GEMM weights on the device: torch's f32 [n_out][c_in][taps] -> bf16 [n_pad][taps * pitch] (tap t of channel c at
// column t * pitch + c, zeros elsewhere) and the bias padded to n_pad.  The ALGORITHMIC work of the weights: padding
// columns / rows (zero weights: view lead-ins of the 'shuffle' layout, 16-channel padding of the 'bins' pieces) are not
// counted -- nnz MACs, the input channels some weight reads (k_real), the output channels some weight or bias produces
// (n_real)
struct GemmWeights { __nv_bfloat16* w = nullptr; float* bias = nullptr; long long nnz = 0; int k_real = 0, n_real = 0; };

int upload_gemm_weights(pifpaf_net* net, const float* weight, const float* bias, int n_out, int c_in, int taps,
                        int pitch, int n_pad, GemmWeights* gw) {
    const size_t ld = (size_t)taps * pitch;
    std::vector<__nv_bfloat16> w((size_t)n_pad * ld, __float2bfloat16(0.f));
    std::vector<float> b(n_pad, 0.f);
    std::vector<char> k_used(c_in, 0);
    *gw = GemmWeights{};
    for (int n = 0; n < n_out; n++) {
        bool row = bias != nullptr && bias[n] != 0.f;
        for (int c = 0; c < c_in; c++)
            for (int t = 0; t < taps; t++) {
                const float v = weight[((size_t)n * c_in + c) * taps + t];
                w[(size_t)n * ld + (size_t)t * pitch + c] = __float2bfloat16(v);
                if (v != 0.f) { gw->nnz++; k_used[c] = 1; row = true; }
            }
        gw->n_real += row ? 1 : 0;
        b[n] = bias ? bias[n] : 0.f;
    }
    for (int c = 0; c < c_in; c++) gw->k_real += k_used[c];
    const int rc = net_upload(net, &gw->w, w);
    return rc != PIFPAF_OK ? rc : net_upload(net, &gw->bias, b);
}

// depthwise weights on the device: torch's f32 [channels][taps] -> tap-major [taps][C], the bias padded to C
int upload_dw_weights(pifpaf_net* net, const float* weight, const float* bias, int channels, int C, int taps,
                      float** d_w, float** d_b) {
    std::vector<float> w((size_t)taps * C, 0.f), b(C, 0.f);
    for (int c = 0; c < channels; c++) {
        for (int t = 0; t < taps; t++) w[(size_t)t * C + c] = weight[(size_t)c * taps + t];
        b[c] = bias ? bias[c] : 0.f;
    }
    const int rc = net_upload(net, d_w, w);
    return rc != PIFPAF_OK ? rc : net_upload(net, d_b, b);
}

// common 1x1 GEMM emit: weights [n_out][k_cols] f32 host -> bf16 [n_pad][k_pad8] device, bias padded
int emit_gemm(pifpaf_net* net, Op& op, int in_tensor, int in_col_off, int k_cols, int n_out,
              const float* weight, const float* bias) {
    const Tensor& tin = net->tensors[in_tensor];
    // a TMA inner coordinate must be 16-byte aligned
    PIFPAF_CHECK_ARG(in_col_off >= 0 && in_col_off % 8 == 0 && in_col_off + k_cols <= tin.c,
                     "conv1x1 input column window must start on a multiple of 8 channels and lie inside the tensor");
    int block_n, n_blocks;
    choose_block_n(n_out, &block_n, &n_blocks);
    const int num_k_blocks = (k_cols + BK - 1) / BK;
    // weights-resident GEMMs stream A through what the resident weight tile leaves of the shared memory: with
    // K = 352..416 and a 176..208-column tile that is 4-5 stages of 16 KB, too few bytes in flight per SM to cover
    // the DRAM latency.  Narrower tiles (more
    // n blocks, A re-read from L2 by each of them) buy the stages back.
    if (net->gemm_res_stages > 0) {
        const int np = pad16(n_out);
        int st = resident_stages(block_n, n_blocks, num_k_blocks, false);
        while (st > 0 && st < net->gemm_res_stages && block_n > 64) {
            const int nb = n_blocks + 1, bn = pad16((np + nb - 1) / nb);
            if (bn < 64) break;
            n_blocks = nb; block_n = bn;
            st = resident_stages(block_n, n_blocks, num_k_blocks, false);
        }
    }
    const int n_pad = block_n * n_blocks;
    const int k_pad = pad8(k_cols);
    GemmWeights gw;
    int rc = upload_gemm_weights(net, weight, bias, n_out, k_cols, 1, k_pad, n_pad, &gw);
    if (rc != PIFPAF_OK) return rc;

    GemmArgs& g = op.g;
    const size_t rows_max = (size_t)net->max_batch * tin.h * tin.w;
    g.N = n_out; g.K = k_cols; g.a_col0 = in_col_off;
    g.block_n = block_n; g.n_blocks = n_blocks;
    g.num_k_blocks = num_k_blocks;
    g.bias = gw.bias;
    g.a = tin.data + in_col_off; g.lda = tin.c; g.wgt = gw.w; g.ldw = k_pad;
    op.a_tensor = in_tensor; op.rows_per_image = tin.h * tin.w;
    op.n_real = gw.n_real;
    op.flops_per_image = 2.0 * (double)op.rows_per_image * (double)gw.nnz;
    op.bytes_per_image = (double)op.rows_per_image * gw.k_real * 2.0;      // A read once (bf16); outputs added by the caller
    op.a_bytes_per_image = op.bytes_per_image;
    op.weight_bytes = (double)gw.nnz * 2.0;
    // the map covers the whole tensor; the view's first column is a TMA coordinate (16-byte aligned).
    // Columns past the view multiply zero weight rows (B is zero padded), columns past the tensor are zero filled.
    rc = make_tmap(&op.tmap_a, tin.data, rows_max, (uint64_t)tin.c, (uint64_t)tin.c, BM);
    if (rc != PIFPAF_OK) return rc;
    rc = make_tmap(&op.tmap_b, gw.w, (uint64_t)n_pad, (uint64_t)k_pad, (uint64_t)k_pad, (uint32_t)block_n);
    return rc;
}

// the residual a plain GEMM epilogue adds: columns [residual_col_off, + N) of an ho x wo tensor
int set_residual(const pifpaf_net* net, GemmArgs& g, int residual_tensor, int residual_col_off, int ho, int wo) {
    PIFPAF_CHECK_ARG(residual_tensor < (int)net->tensors.size(), "bad residual tensor");
    const Tensor& tr = net->tensors[residual_tensor];
    PIFPAF_CHECK_ARG(tr.h == ho && tr.w == wo && residual_col_off % 8 == 0 && residual_col_off + g.N <= tr.c,
                     "residual tensor shape mismatch");
    g.res = tr.data; g.ld_res = tr.c; g.res_col_off = residual_col_off;
    return PIFPAF_OK;
}

// plain 1x1 GEMM epilogue into the window [out_col_off, + pad8(N)) of `to`: with a residual (residual_tensor >= 0)
// the per-lane epilogue adds it, without one the TMA-store epilogue writes the window.
// ReLU6 GEMMs keep the per-lane epilogue: a ReLU6 clamp in the TMA-store epilogue (a uniform branch per fragment
// group) slowed the ShuffleNetV2K forward, which never uses it, by 0.15 ms of 24.7 (64 images at 641 px, H100)
int set_plain_epilogue(const pifpaf_net* net, Op& op, int relu, const Tensor& to, int out_col_off,
                       int residual_tensor, int residual_col_off) {
    GemmArgs& g = op.g;
    g.mode = MODE_PLAIN; g.relu = relu; g.out = to.data; g.ldo = to.c; g.out_col_off = out_col_off;
    op.bytes_per_image += (double)op.rows_per_image * op.n_real * 2.0 * (residual_tensor >= 0 ? 2.0 : 1.0);
    if (residual_tensor >= 0) return set_residual(net, g, residual_tensor, residual_col_off, to.h, to.w);
    if (net->gemm_tma_store && g.relu != ACT_RELU6) {
        g.tma_store = 1;
        op.store_views = {Op::StoreView{to.data + g.out_col_off, pad8(g.N), to.c}};
    }
    return PIFPAF_OK;
}

// destination table of a scatter epilogue, uploaded: the pieces tile [0, n_out) in order, in multiples of 16 columns;
// piece i lands in the columns [piece_tensor_col[i], + piece_count[i]) of tensor piece_tensor[i] (h x w pixels).
// Entry j covers the 16 columns from 16 j: base, row pitch and `store` = (store map << 16) | first column, for the
// TMA-store epilogue with one store map per destination tensor (map_tensor, in order of first use)
int upload_dest_groups(pifpaf_net* net, int n_pad, int n_out, int h, int w, int n_pieces, const int32_t* piece_col0,
                       const int32_t* piece_count, const int32_t* piece_tensor, const int32_t* piece_tensor_col,
                       const DestGroup** d_groups, std::vector<int>* map_tensor) {
    std::vector<DestGroup> groups((size_t)n_pad / 16, DestGroup{nullptr, 0, 0});
    map_tensor->clear();
    int expect = 0;
    for (int i = 0; i < n_pieces; i++) {
        PIFPAF_CHECK_ARG(piece_col0[i] == expect && piece_count[i] >= 16 && piece_count[i] % 16 == 0,
                         "pieces must tile [0, n_out) in order, in multiples of 16 columns");
        PIFPAF_CHECK_ARG(piece_tensor[i] >= 0 && piece_tensor[i] < (int)net->tensors.size(), "bad piece tensor id");
        const Tensor& to = net->tensors[piece_tensor[i]];
        PIFPAF_CHECK_ARG(to.h == h && to.w == w, "a piece tensor must have the output's spatial shape");
        PIFPAF_CHECK_ARG(piece_tensor_col[i] >= 0 && piece_tensor_col[i] % 16 == 0 &&
                         piece_tensor_col[i] + piece_count[i] <= to.c, "piece window outside its tensor");
        int mi = 0;
        while (mi < (int)map_tensor->size() && (*map_tensor)[mi] != piece_tensor[i]) mi++;
        if (mi == (int)map_tensor->size()) map_tensor->push_back(piece_tensor[i]);
        for (int c = 0; c < piece_count[i]; c += 16)
            groups[(size_t)(expect + c) / 16] = DestGroup{to.data + piece_tensor_col[i] + c, to.c,
                                                          (mi << 16) | (piece_tensor_col[i] + c)};
        expect += piece_count[i];
    }
    PIFPAF_CHECK_ARG(expect == n_out, "pieces must cover all n_out columns");
    DestGroup* d = nullptr;
    const int rc = net_upload(net, &d, groups);
    *d_groups = d;
    return rc;
}

// The kernels of a depthwise op, chosen once at emit; launch_dw only reads them.  TMA route (gemm_impl 0): a DW_TMA
// entry and the shared memory of its launch.  SIMT route (gemm_impl 1, or no TMA entry): k_dwconv5<S> or k_dwconv.
void choose_dw_kernels(const pifpaf_net* net, Op& op) {
    const DwArgs& a = op.dw;
    const int kernel = a.kernel, stride = a.stride, relu = a.relu, dilation = op.dw_dil;
    if (dilation == 2 && kernel == 5 && stride == 1 && relu != ACT_RELU6) {
        op.dw_tma = &DW_TMA[DW_K5_S1_D2];
    } else if (dilation == 1 && (kernel == 3 || (kernel == 5 && relu != ACT_RELU6)) && (stride == 1 || stride == 2)) {
        op.dw_tma = &DW_TMA[kernel == 3 ? (stride == 1 ? DW_K3_S1 : DW_K3_S2) : (stride == 1 ? DW_K5_S1 : DW_K5_S2)];
    }
    if (op.dw_tma) op.smem = op.dw_tma->smem;
    // channel-block-fastest order with the weights staged in shared memory while they fit
    const size_t smem_cf = op.smem + (size_t)26 * a.C8 * 8 * sizeof(float);
    if (op.dw_tma == &DW_TMA[DW_K5_S2] && net->dw_cbf && (a.C8 + 7) / 8 > 1 &&
        smem_cf <= (size_t)DW_TMA[DW_K5_S2_CBF].smem) {
        op.dw_tma = &DW_TMA[DW_K5_S2_CBF];
        op.smem = smem_cf;
    }
    if (kernel == 5 && dilation == 1 && (stride == 1 || stride == 2))
        op.dw_simt5 = stride == 1 ? k_dwconv5<1> : k_dwconv5<2>;
}

// Decides, once all ops are known, which 1x1 GEMM -> depthwise pairs run as one k_pw_dw launch.  The GEMM qualifies
// when it is plain (no residual, shuffle or implicit conv), reads one K block from column 0 of a tensor of at most
// PWDW_K channels and writes column 0 of its output tensor; it is fused when the next op is the TMA depthwise 5x5,
// stride 2, pad 2 (in either item order) reading that tensor from column 0, and no other op touches the tensor.
int plan_pw_dw(pifpaf_net* net) {
    net->pw_dw_planned = net->ops.size();
    for (Op& op : net->ops) { op.elided = false; op.pw_dw = false; }
    if (!net->fuse_pw_dw) return PIFPAF_OK;
    for (size_t i = 0; i + 1 < net->ops.size(); i++) {
        Op& gop = net->ops[i];
        Op& dop = net->ops[i + 1];
        const GemmArgs& g = gop.g;
        const DwArgs& d = dop.dw;
        if (gop.kind != OP_GEMM || dop.kind != OP_DW || !dop.dw_tma || d.kernel != 5 || d.stride != 2) continue;
        if (g.mode != MODE_PLAIN || g.conv_k != 0 || g.res != nullptr || g.num_k_blocks != 1 || g.a_col0 != 0 ||
            g.out_col_off != 0 || g.relu == ACT_RELU6)
            continue;
        // k_pw_dw is built for the 5x5 stride-2 depthwise conv (DW_K5_S2: ReLU at most, not MobileNetV2's 3x3 + ReLU6 pairs)
        if (d.pad != 2 || d.in != g.out || d.in_col_off != 0) continue;
        const Tensor& tin = net->tensors[gop.a_tensor];
        if (tin.c > PWDW_K) continue;
        int t_mid = -1;
        for (int t = 0; t < (int)net->tensors.size(); t++)
            if (net->tensors[t].data == g.out) t_mid = t;
        bool private_mid = t_mid >= 0;
        for (size_t j = 0; j < net->ops.size() && private_mid; j++)
            if (j != i && j != i + 1)
                for (int t : net->ops[j].touches) private_mid = private_mid && t != t_mid;
        const int cblks = (d.C8 + 7) / 8;
        const size_t smem = pw_dw_smem_bytes(PwDwS2::IN_BYTES, PwDwS2::MID_BYTES, cblks, d.C8 * 8);
        if (!private_mid || smem > 226 * 1024) continue;
        PwDwArgs& p = dop.pw;
        p.dw = d;
        p.w1 = g.wgt; p.ldw1 = g.ldw; p.n1 = g.block_n * g.n_blocks; p.b1 = g.bias; p.relu1 = g.relu;
        p.Hin = tin.h; p.Win = tin.w; p.cblks = cblks;
        const int rc = make_tmap_dw(&dop.tmap_pw, tin.data, (uint64_t)tin.c, (uint64_t)tin.w, (uint64_t)tin.h,
                                    (uint64_t)net->max_batch, (uint64_t)tin.c, PwDwS2::IW, PwDwS2::IH, PWDW_K,
                                    CU_TENSOR_MAP_SWIZZLE_64B);
        if (rc != PIFPAF_OK) return rc;
        dop.pw_smem = smem;
        // both ops' FLOPs; the 1x1 input read once, the depthwise output written once, the 1x1 weights
        dop.pw_flops_per_image = gop.flops_per_image + dop.flops_per_image;
        dop.pw_bytes_per_image = gop.a_bytes_per_image + dop.dw_out_bytes_per_image;
        dop.pw_weight_bytes = gop.weight_bytes + dop.weight_bytes;
        gop.elided = true;
        dop.pw_dw = true;
    }
    return PIFPAF_OK;
}

int effective_sms(const pifpaf_net* net) { return net->sm_limit > 0 ? std::min(net->sm_limit, net->n_sm) : net->n_sm; }

// one launch of a GEMM op (k_gemm_wg, or the SIMT debug kernel for gemm_impl == 1) at this batch
int launch_gemm(pifpaf_net* net, Op& op, int batch, int gemm_impl, bool pdl, cudaStream_t st) {
    const int n_sm = effective_sms(net);
    GemmArgs g = op.g;
    if (g.mode == MODE_HEADS)
        for (int i = 0; i < net->n_heads; i++) g.head_base[i] = net->head_out[net->head_cur][i];
    g.M = batch * op.rows_per_image;
    g.m_blocks = g.conv_k > 0 ? batch * op.tiles_per_image : (g.M + BM - 1) / BM;
    if (gemm_impl == 1) {
        const long long jobs = (long long)g.m_blocks * 4 * (g.n_blocks * g.block_n / CHUNK);
        const int grid = (int)std::min<long long>((jobs + 3) / 4, (long long)n_sm * 16);
        return launch_k(false, k_gemm_simt, dim3(grid), dim3(128), 0, st, g);
    }
    int grid = std::min(g.m_blocks * g.n_blocks, n_sm);
    if (g.b_resident) grid = std::max(1, std::min(n_sm / g.n_blocks, g.m_blocks)) * g.n_blocks;
    if (g.tma_store && op.store_rows != g.M) {
        for (size_t i = 0; i < op.store_views.size(); i++) {
            const Op::StoreView& v = op.store_views[i];
            const int rc = make_tmap_store(&op.smaps.m[i], v.base, (uint64_t)g.M, (uint64_t)v.cols, (uint64_t)v.ld);
            if (rc != PIFPAF_OK) return rc;
        }
        op.store_rows = g.M;
    }
    auto* kern = GEMM_KERNELS[tile_groups(g.block_n)][tile_last(g.block_n)];
    return launch_k(pdl, kern, dim3(grid), dim3(GEMM_THREADS), op.smem, st, op.tmap_a, op.tmap_b,
                    g.src_tma ? op.tmap_src : op.tmap_a, op.smaps, g);
}

struct RawImages { const uint8_t* images; float mean[3], stdev[3]; };

// the stem, on the f32 images or on the raw uint8 ones (u8).  Always the first op, so launched without PDL
int launch_input_conv(const pifpaf_net* net, const Op& op, int batch, const float* images, const RawImages* u8,
                      cudaStream_t st) {
    InConvArgs a = op.ic;
    a.in = images; a.B = batch;
    const long long total = (long long)batch * a.Hout * a.Wout;
    const int grid = (int)std::min<long long>((total + 255) / 256, (long long)effective_sms(net) * 16);
    if (u8 != nullptr) {
        a.in_u8 = u8->images;
        for (int c = 0; c < 3; c++) { a.mean[c] = u8->mean[c]; a.stdev[c] = u8->stdev[c]; }
    }
    return launch_k(false, INPUT_CONV_KERNELS[u8 != nullptr][a.kernel / 2], dim3(grid), dim3(256),
                    input_conv_smem_bytes(a.kernel, a.C8), st, a);
}

// the fused depthwise -> 1x1 op (k_dw_gemm)
int launch_dw_gemm(const pifpaf_net* net, const Op& op, int batch, int gemm_impl, bool pdl, cudaStream_t st) {
    PIFPAF_CHECK_ARG(gemm_impl == 0, "the fused depthwise -> 1x1 op has no SIMT debug variant (compile the net with fuse_dw=False)");
    GemmArgs g = op.g;
    g.M = batch * op.rows_per_image;
    g.m_blocks = batch * op.tiles_per_image;
    const int grid = std::max(1, std::min(effective_sms(net) / g.n_blocks, g.m_blocks)) * g.n_blocks;
    auto* kern = DW_GEMM_KERNELS[tile_groups(g.block_n)][tile_last(g.block_n)];
    return launch_k(pdl, kern, dim3(grid), dim3(FD_THREADS), op.smem, st, op.tmap_dw, op.tmap_b, g, op.fu);
}

// a depthwise op: k_pw_dw when plan_pw_dw paired it with the 1x1 before it, else the route choose_dw_kernels stored.
// k_dwconv5 and k_dwconv run no griddepcontrol.wait, so they launch without PDL
int launch_dw(const pifpaf_net* net, const Op& op, int batch, int gemm_impl, bool pdl, cudaStream_t st) {
    const int n_sm = effective_sms(net);
    DwArgs a = op.dw;
    a.B = batch;
    if (op.pw_dw && gemm_impl == 0) {
        PwDwArgs p = op.pw;
        p.dw.B = batch;
        const long long total = (long long)batch * ((a.Hout + PWDW_TH - 1) / PWDW_TH) * ((a.Wout + PWDW_TW - 1) / PWDW_TW);
        const int grid = (int)std::min<long long>(total, (long long)n_sm);     // 1 CTA per SM by shared memory
        return launch_k(pdl, k_pw_dw<2, PWDW_TH, PWDW_TW, PWDW_BW>, dim3(grid), dim3(PwDwS2::THREADS), op.pw_smem, st,
                        op.tmap_pw, p);
    }
    if (op.dw_tma && gemm_impl == 0) {
        const DwTmaVariant* v = op.dw_tma;
        const long long total = (long long)batch * ((a.Hout + v->th - 1) / v->th) * ((a.Wout + v->tw - 1) / v->tw) *
                                ((a.C8 + 7) / 8);
        const int grid = (int)std::min<long long>(total, (long long)n_sm * v->ctas_per_sm);
        return launch_k(pdl, v->kernel, dim3(grid), dim3(v->threads), op.smem, st, op.tmap_dw, a);
    }
    if (op.dw_simt5) {
        const long long total = (long long)batch * ((a.Hout + DW_OY - 1) / DW_OY) * DW_OY *
                                ((a.Wout + DW_OX - 1) / DW_OX) * a.C8;
        const int grid = (int)std::min<long long>((total + 255) / 256, (long long)n_sm * 64);
        return launch_k(false, op.dw_simt5, dim3(grid), dim3(256), 0, st, a);
    }
    const long long total = (long long)batch * a.Hout * a.Wout * a.C8;
    const int grid = (int)std::min<long long>((total + 255) / 256, (long long)n_sm * 32);
    return launch_k(false, k_dwconv, dim3(grid), dim3(256), 0, st, a, op.dw_dil);
}

int launch_maxpool(const pifpaf_net* net, const Op& op, int batch, bool pdl, cudaStream_t st) {
    DwArgs a = op.dw;
    a.B = batch;
    const long long total = (long long)batch * a.Hout * a.Wout * a.C8;
    const int grid = (int)std::min<long long>((total + 255) / 256, (long long)effective_sms(net) * 32);
    return launch_k(pdl, k_maxpool, dim3(grid), dim3(256), 0, st, a);
}

int launch_op(pifpaf_net* net, Op& op, int batch, int gemm_impl, bool pdl, cudaStream_t st, const float* images,
              const RawImages* u8) {
    switch (op.kind) {
    case OP_INPUT_CONV: return launch_input_conv(net, op, batch, images, u8, st);
    case OP_DW: return launch_dw(net, op, batch, gemm_impl, pdl, st);
    case OP_FUSED: return launch_dw_gemm(net, op, batch, gemm_impl, pdl, st);
    case OP_MAXPOOL: return launch_maxpool(net, op, batch, pdl, st);
    default: return launch_gemm(net, op, batch, gemm_impl, pdl, st);
    }
}

}  // namespace

extern "C" {

int pifpaf_net_create(pifpaf_net_t** out, int32_t device, int32_t max_batch) {
    PIFPAF_CHECK_ARG(out != nullptr, "out is null");
    *out = nullptr;
    PIFPAF_CHECK_ARG(max_batch >= 1, "max_batch must be >= 1");
    int n_dev = 0;
    PIFPAF_CUDA_TRY(cudaGetDeviceCount(&n_dev));
    PIFPAF_CHECK_ARG(device >= 0 && device < n_dev, "no such CUDA device");
    PIFPAF_CUDA_TRY(cudaSetDevice(device));
    cudaDeviceProp prop;
    PIFPAF_CUDA_TRY(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9) {
        pifpaf::set_error("libpifpaf_b200 is built for sm_90a only; device %d is sm_%d%d", device, prop.major, prop.minor);
        return PIFPAF_E_CUDA;
    }
    pifpaf_net* net = new pifpaf_net();
    net->device = device; net->max_batch = max_batch; net->n_sm = prop.multiProcessorCount;
    if (const char* e = std::getenv("PIFPAF_DW_CBF")) net->dw_cbf = std::atoi(e) != 0;
    if (const char* e = std::getenv("PIFPAF_PDL")) net->pdl = std::atoi(e) != 0;
    if (const char* e = std::getenv("PIFPAF_GEMM_RES_STAGES")) net->gemm_res_stages = std::atoi(e);
    if (const char* e = std::getenv("PIFPAF_GEMM_TMA_STORE")) net->gemm_tma_store = std::atoi(e) != 0;
    if (const char* e = std::getenv("PIFPAF_FUSE_PW_DW")) net->fuse_pw_dw = std::atoi(e) != 0;
    // the shared-memory limit of every kernel the forward launches with more than the default 48 KB, from the tables the
    // launches index (the stem stages its weights: 7x7 with more than 72 channels is past 48 KB)
    PIFPAF_CUDA_TRY(cudaFuncSetAttribute(k_pw_dw<2, PWDW_TH, PWDW_TW, PWDW_BW>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         226 * 1024));
    for (auto& row : GEMM_KERNELS)
        for (auto* k : row) PIFPAF_CUDA_TRY(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, 226 * 1024));
    for (auto& row : DW_GEMM_KERNELS)
        for (auto* k : row) PIFPAF_CUDA_TRY(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, 226 * 1024));
    for (const DwTmaVariant& v : DW_TMA)
        PIFPAF_CUDA_TRY(cudaFuncSetAttribute(v.kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, v.smem));
    for (auto& row : INPUT_CONV_KERNELS)
        for (auto* k : row) PIFPAF_CUDA_TRY(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, INCONV_SMEM_MAX));
    *out = net;
    return PIFPAF_OK;
}

void pifpaf_net_destroy(pifpaf_net_t* net) {
    if (!net) return;
    cudaSetDevice(net->device);
    for (void* p : net->owned) cudaFree(p);
    delete net;
}

int pifpaf_net_tensor(pifpaf_net_t* net, int32_t h, int32_t w, int32_t c_phys, int32_t* id) {
    PIFPAF_CHECK_ARG(net != nullptr && id != nullptr, "null argument");
    PIFPAF_CHECK_ARG(h >= 1 && w >= 1 && c_phys >= 16 && c_phys % 16 == 0, "tensor shape: c_phys must be a multiple of 16");
    PIFPAF_CUDA_TRY(cudaSetDevice(net->device));
    Tensor t; t.h = h; t.w = w; t.c = c_phys; t.data = nullptr;
    // + one tile of slack rows so that TMA boxes of the last partial M tile stay in mapped memory
    int rc = net_alloc(net, &t.data, ((size_t)net->max_batch * h * w + BM) * c_phys, true);
    if (rc != PIFPAF_OK) return rc;
    net->tensors.push_back(t);
    *id = (int)net->tensors.size() - 1;
    return PIFPAF_OK;
}

int pifpaf_net_input_conv(pifpaf_net_t* net, int32_t in_h, int32_t in_w, int32_t kernel, int32_t stride,
                          int32_t pad, int32_t c_out, const float* weight, const float* bias,
                          int32_t relu, int32_t out_tensor) {
    PIFPAF_CHECK_ARG(net != nullptr && weight != nullptr, "null argument");
    PIFPAF_CHECK_ARG(out_tensor >= 0 && out_tensor < (int)net->tensors.size(), "bad tensor id");
    PIFPAF_CHECK_ARG(relu >= ACT_NONE && relu <= ACT_RELU6, "activation code must be 0 (none), 1 (ReLU) or 2 (ReLU6)");
    const Tensor& to = net->tensors[out_tensor];
    const int ho = (in_h + 2 * pad - kernel) / stride + 1, wo = (in_w + 2 * pad - kernel) / stride + 1;
    PIFPAF_CHECK_ARG(to.h == ho && to.w == wo && to.c >= pad8(c_out), "output tensor shape mismatch");
    PIFPAF_CHECK_ARG(kernel == 1 || kernel == 3 || kernel == 5 || kernel == 7, "input conv kernel must be 1, 3, 5 or 7");
    PIFPAF_CHECK_ARG(c_out >= 1 && input_conv_smem_bytes(kernel, pad8(c_out) / 8) <= (size_t)INCONV_SMEM_MAX,
                     "input conv: the weights of a kxk conv with this many output channels do not fit in shared memory");
    PIFPAF_CUDA_TRY(cudaSetDevice(net->device));
    const int C = pad8(c_out);
    std::vector<float> w((size_t)3 * kernel * kernel * C, 0.f), b(C, 0.f);
    for (int co = 0; co < c_out; co++) {
        for (int ci = 0; ci < 3; ci++)
            for (int ky = 0; ky < kernel; ky++)
                for (int kx = 0; kx < kernel; kx++)
                    w[(size_t)((ci * kernel + ky) * kernel + kx) * C + co] =
                        weight[(((size_t)co * 3 + ci) * kernel + ky) * kernel + kx];
        b[co] = bias ? bias[co] : 0.f;
    }
    Op op; op.kind = OP_INPUT_CONV;
    float *d_w = nullptr, *d_b = nullptr;
    int rc = net_upload(net, &d_w, w); if (rc != PIFPAF_OK) return rc;
    rc = net_upload(net, &d_b, b); if (rc != PIFPAF_OK) return rc;
    InConvArgs& a = op.ic;
    a.in = nullptr; a.out = to.data; a.ld_out = to.c; a.weight = d_w; a.bias = d_b;
    a.Hin = in_h; a.Win = in_w; a.Hout = ho; a.Wout = wo; a.C8 = C / 8;
    a.kernel = kernel; a.stride = stride; a.pad = pad; a.relu = relu;
    op.flops_per_image = 2.0 * ho * wo * c_out * 3.0 * kernel * kernel;
    op.bytes_per_image = (double)in_h * in_w * 3 * 4.0 + (double)ho * wo * c_out * 2.0;
    op.touches = {out_tensor};
    net->in_h = in_h; net->in_w = in_w;
    net->ops.push_back(op);
    return PIFPAF_OK;
}

int pifpaf_net_conv1x1(pifpaf_net_t* net, int32_t in_tensor, int32_t in_col_off, int32_t k_cols,
                       int32_t n_out, const float* weight, const float* bias, int32_t relu,
                       int32_t out_tensor, int32_t out_col_off,
                       int32_t shuffle_src_tensor, int32_t shuffle_src_col_off) {
    PIFPAF_CHECK_ARG(net != nullptr && weight != nullptr, "null argument");
    const int nt = (int)net->tensors.size();
    PIFPAF_CHECK_ARG(in_tensor >= 0 && in_tensor < nt && out_tensor >= 0 && out_tensor < nt, "bad tensor id");
    PIFPAF_CHECK_ARG(k_cols >= 1 && n_out >= 1, "bad conv size");
    PIFPAF_CHECK_ARG(relu == ACT_NONE || relu == ACT_RELU || (relu == ACT_RELU6 && shuffle_src_tensor < 0),
                     "activation code must be 0 (none), 1 (ReLU) or 2 (ReLU6); the shuffle epilogue takes 0 or 1");
    PIFPAF_CUDA_TRY(cudaSetDevice(net->device));
    const Tensor& tin = net->tensors[in_tensor];
    const Tensor& to = net->tensors[out_tensor];
    PIFPAF_CHECK_ARG(tin.h == to.h && tin.w == to.w, "conv1x1 keeps the spatial shape");
    Op op; op.kind = OP_GEMM;
    int rc = emit_gemm(net, op, in_tensor, in_col_off, k_cols, n_out, weight, bias);
    if (rc != PIFPAF_OK) return rc;
    GemmArgs& g = op.g;
    PIFPAF_CHECK_ARG(out_col_off % 16 == 0, "output column offset must be a multiple of 16");
    if (shuffle_src_tensor < 0) {
        PIFPAF_CHECK_ARG(out_col_off + pad8(n_out) <= to.c, "output window outside the tensor");
        rc = set_plain_epilogue(net, op, relu, to, out_col_off, -1, 0);
        if (rc != PIFPAF_OK) return rc;
    } else {
        PIFPAF_CHECK_ARG(shuffle_src_tensor < nt, "bad shuffle source tensor");
        const Tensor& ts = net->tensors[shuffle_src_tensor];
        PIFPAF_CHECK_ARG(ts.h == to.h && ts.w == to.w, "shuffle source shape mismatch");
        PIFPAF_CHECK_ARG(n_out % 2 == 0, "fused channel_shuffle needs an even branch width");
        PIFPAF_CHECK_ARG(shuffle_src_col_off % 8 == 0 && shuffle_src_col_off + pad16(n_out) <= ts.c + 8,
                         "shuffle source window");
        PIFPAF_CHECK_ARG(out_col_off == 0 && to.c >= 2 * n_out, "shuffle output tensor must hold 2*n_out channels");
        g.mode = MODE_SHUFFLE; g.relu = relu; g.out = to.data; g.ldo = to.c; g.out_col_off = out_col_off;
        // outputs: n_out bf16 per row, and the pass-through half read and re-written
        op.bytes_per_image += (double)op.rows_per_image * op.n_real * 2.0 * 3.0;
        g.src0 = ts.data; g.ld0 = ts.c; g.src0_col_off = shuffle_src_col_off;
        g.half = n_out; g.gap = 0;
        g.src_tma = gemm_smem_bytes(g.block_n, g.n_blocks, 2, true) <= GEMM_SMEM_BUDGET ? 1 : 0;
        // pass-through tile [BM rows][block_n cols], dense rows in shared memory (no swizzle)
        rc = make_tmap_plain(&op.tmap_src, ts.data + shuffle_src_col_off, (uint64_t)net->max_batch * ts.h * ts.w,
                             (uint64_t)std::min(ts.c - shuffle_src_col_off, pad16(n_out)), (uint64_t)ts.c,
                             (uint32_t)g.block_n, BM);
        if (rc != PIFPAF_OK) return rc;
    }
    plan_gemm_smem(op);
    op.touches = {in_tensor, out_tensor, shuffle_src_tensor};
    net->ops.push_back(op);
    return PIFPAF_OK;
}

int pifpaf_net_conv1x1_scatter(pifpaf_net_t* net, int32_t in_tensor, int32_t in_col_off, int32_t k_cols,
                               int32_t n_out, const float* weight, const float* bias, int32_t relu,
                               int32_t n_pieces, const int32_t* piece_col0, const int32_t* piece_count,
                               const int32_t* piece_tensor, const int32_t* piece_tensor_col) {
    PIFPAF_CHECK_ARG(net != nullptr && weight != nullptr && piece_col0 && piece_count && piece_tensor && piece_tensor_col,
                     "null argument");
    const int nt = (int)net->tensors.size();
    PIFPAF_CHECK_ARG(in_tensor >= 0 && in_tensor < nt, "bad tensor id");
    PIFPAF_CHECK_ARG(k_cols >= 1 && n_out >= 16 && n_out % 16 == 0 && n_pieces >= 1, "bad conv size");
    PIFPAF_CHECK_ARG(relu == ACT_NONE || relu == ACT_RELU, "the scatter epilogue takes activation codes 0 (none) and 1 (ReLU)");
    PIFPAF_CUDA_TRY(cudaSetDevice(net->device));
    const Tensor& tin = net->tensors[in_tensor];
    Op op; op.kind = OP_GEMM;
    int rc = emit_gemm(net, op, in_tensor, in_col_off, k_cols, n_out, weight, bias);
    if (rc != PIFPAF_OK) return rc;
    GemmArgs& g = op.g;
    g.mode = MODE_SCATTER; g.relu = relu;
    std::vector<int> map_tensor;
    rc = upload_dest_groups(net, g.n_blocks * g.block_n, n_out, tin.h, tin.w, n_pieces, piece_col0, piece_count,
                            piece_tensor, piece_tensor_col, &g.dest, &map_tensor);
    if (rc != PIFPAF_OK) return rc;
    // TMA-store epilogue: one store map per destination tensor (a chunk's box covers exactly its 16 columns); more
    // destination tensors than store maps: the per-lane store epilogue
    if (net->gemm_tma_store && (int)map_tensor.size() <= MAX_STORE_MAPS) {
        g.tma_store = 1;
        for (int t : map_tensor) {
            const Tensor& to = net->tensors[t];
            op.store_views.push_back(Op::StoreView{to.data, to.c, to.c});
        }
    }
    op.bytes_per_image += (double)op.rows_per_image * op.n_real * 2.0;
    plan_gemm_smem(op);
    op.touches.assign(piece_tensor, piece_tensor + n_pieces);
    op.touches.push_back(in_tensor);
    net->ops.push_back(op);
    return PIFPAF_OK;
}

int pifpaf_net_conv(pifpaf_net_t* net, int32_t in_tensor, int32_t in_col_off, int32_t c_in,
                    int32_t kernel, int32_t stride, int32_t pad, int32_t n_out, const float* weight,
                    const float* bias, int32_t relu, int32_t out_tensor, int32_t out_col_off,
                    int32_t residual_tensor, int32_t residual_col_off) {
    return pifpaf_net_conv_dilated(net, in_tensor, in_col_off, c_in, kernel, stride, pad, n_out, weight, bias, relu,
                                   out_tensor, out_col_off, residual_tensor, residual_col_off, 1);
}

int pifpaf_net_conv_dilated(pifpaf_net_t* net, int32_t in_tensor, int32_t in_col_off, int32_t c_in,
                            int32_t kernel, int32_t stride, int32_t pad, int32_t n_out, const float* weight,
                            const float* bias, int32_t relu, int32_t out_tensor, int32_t out_col_off,
                            int32_t residual_tensor, int32_t residual_col_off, int32_t dilation) {
    PIFPAF_CHECK_ARG(net != nullptr && weight != nullptr, "null argument");
    const int nt = (int)net->tensors.size();
    PIFPAF_CHECK_ARG(in_tensor >= 0 && in_tensor < nt && out_tensor >= 0 && out_tensor < nt, "bad tensor id");
    PIFPAF_CHECK_ARG(kernel >= 1 && kernel <= 7 && stride >= 1 && stride <= 2 && pad >= 0, "unsupported conv geometry");
    PIFPAF_CHECK_ARG(dilation >= 1 && dilation <= 64, "conv dilation must be 1 to 64");
    PIFPAF_CHECK_ARG(relu >= ACT_NONE && relu <= ACT_RELU6, "activation code must be 0 (none), 1 (ReLU) or 2 (ReLU6)");
    // the stride-2 tensor map steps over every other input pixel; dilated taps would need their own traversal
    PIFPAF_CHECK_ARG(dilation == 1 || stride == 1, "a dilated conv (dilation > 1) must have stride 1");
    PIFPAF_CHECK_ARG(c_in >= 1 && n_out >= 1, "bad conv size");
    PIFPAF_CUDA_TRY(cudaSetDevice(net->device));
    const Tensor& tin = net->tensors[in_tensor];
    const Tensor& to = net->tensors[out_tensor];
    const int span = dilation * (kernel - 1) + 1;
    PIFPAF_CHECK_ARG(tin.h + 2 * pad >= span && tin.w + 2 * pad >= span, "conv window larger than the padded input");
    const int ho = (tin.h + 2 * pad - span) / stride + 1, wo = (tin.w + 2 * pad - span) / stride + 1;
    PIFPAF_CHECK_ARG(to.h == ho && to.w == wo, "conv output tensor shape mismatch");
    PIFPAF_CHECK_ARG(in_col_off % 8 == 0 && in_col_off + c_in <= tin.c, "conv input column window");
    PIFPAF_CHECK_ARG(out_col_off % 16 == 0 && out_col_off + pad8(n_out) <= to.c, "conv output column window");
    if (kernel == 1 && stride == 1 && pad == 0) {
        // pointwise: the flat [pixels x channels] GEMM (no patch tiling waste), residual fused the same way
        Op op; op.kind = OP_GEMM;
        int rc = emit_gemm(net, op, in_tensor, in_col_off, c_in, n_out, weight, bias);
        if (rc != PIFPAF_OK) return rc;
        rc = set_plain_epilogue(net, op, relu, to, out_col_off, residual_tensor, residual_col_off);
        if (rc != PIFPAF_OK) return rc;
        plan_gemm_smem(op);
        op.touches = {in_tensor, out_tensor, residual_tensor};
        net->ops.push_back(op);
        return PIFPAF_OK;
    }
    Op op; op.kind = OP_GEMM;
    int block_n, n_blocks;
    choose_block_n(n_out, &block_n, &n_blocks);
    const int n_pad = block_n * n_blocks;
    const int taps = kernel * kernel, cblocks = (c_in + BK - 1) / BK;
    const int k_total = taps * cblocks * BK;
    // bf16 [n_pad][tap][cblocks*64]
    GemmWeights gw;
    int rc = upload_gemm_weights(net, weight, bias, n_out, c_in, taps, cblocks * BK, n_pad, &gw);
    if (rc != PIFPAF_OK) return rc;
    GemmArgs& g = op.g;
    g.N = n_out; g.K = c_in;
    g.block_n = block_n; g.n_blocks = n_blocks;
    g.num_k_blocks = taps * cblocks;
    g.bias = gw.bias; g.mode = MODE_PLAIN; g.relu = relu;
    g.out = to.data; g.ldo = to.c; g.out_col_off = out_col_off;
    g.conv_k = kernel; g.conv_stride = stride; g.conv_pad = pad; g.conv_dil = dilation; g.conv_cblocks = cblocks;
    g.Hi = tin.h; g.Wi = tin.w; g.Ho = ho; g.Wo = wo;
    g.tiles_x = (wo + PW - 1) / PW; g.tiles_y = (ho + PH - 1) / PH;
    g.a = tin.data + in_col_off; g.lda = tin.c; g.wgt = gw.w; g.ldw = k_total;
    if (residual_tensor >= 0) {
        rc = set_residual(net, g, residual_tensor, residual_col_off, ho, wo);
        if (rc != PIFPAF_OK) return rc;
    }
    op.a_tensor = in_tensor; op.rows_per_image = ho * wo; op.tiles_per_image = g.tiles_x * g.tiles_y;
    plan_gemm_smem(op);
    // dense shapes: every weight and input channel counted
    op.flops_per_image = 2.0 * (double)ho * wo * n_out * c_in * taps;
    op.bytes_per_image = (double)tin.h * tin.w * c_in * 2.0 + (double)ho * wo * n_out * 2.0 * (residual_tensor >= 0 ? 2.0 : 1.0);
    op.weight_bytes = (double)n_out * c_in * taps * 2.0;
    rc = make_tmap_conv(&op.tmap_a, tin.data + in_col_off, (uint64_t)c_in, (uint64_t)tin.w, (uint64_t)tin.h,
                        (uint64_t)net->max_batch, (uint64_t)tin.c, stride);
    if (rc != PIFPAF_OK) return rc;
    rc = make_tmap(&op.tmap_b, gw.w, (uint64_t)n_pad, (uint64_t)k_total, (uint64_t)k_total, (uint32_t)block_n);
    if (rc != PIFPAF_OK) return rc;
    op.touches = {in_tensor, out_tensor, residual_tensor};
    net->ops.push_back(op);
    return PIFPAF_OK;
}

int pifpaf_net_dwconv(pifpaf_net_t* net, int32_t in_tensor, int32_t in_col_off, int32_t channels,
                      int32_t kernel, int32_t stride, int32_t pad, const float* weight, const float* bias,
                      int32_t relu, int32_t out_tensor, int32_t out_col_off) {
    return pifpaf_net_dwconv_dilated(net, in_tensor, in_col_off, channels, kernel, stride, pad, weight, bias, relu,
                                     out_tensor, out_col_off, 1);
}

int pifpaf_net_dwconv_dilated(pifpaf_net_t* net, int32_t in_tensor, int32_t in_col_off, int32_t channels,
                              int32_t kernel, int32_t stride, int32_t pad, const float* weight, const float* bias,
                              int32_t relu, int32_t out_tensor, int32_t out_col_off, int32_t dilation) {
    PIFPAF_CHECK_ARG(net != nullptr && weight != nullptr, "null argument");
    const int nt = (int)net->tensors.size();
    PIFPAF_CHECK_ARG(in_tensor >= 0 && in_tensor < nt && out_tensor >= 0 && out_tensor < nt, "bad tensor id");
    PIFPAF_CHECK_ARG(relu >= ACT_NONE && relu <= ACT_RELU6, "activation code must be 0 (none), 1 (ReLU) or 2 (ReLU6)");
    PIFPAF_CHECK_ARG(dilation >= 1, "dwconv dilation must be at least 1");
    // the reference pairs dilation with stride 1 (basenetworks.py:297-306); the tiled kernels assume it
    PIFPAF_CHECK_ARG(dilation == 1 || stride == 1, "a dilated dwconv (dilation > 1) must have stride 1");
    const Tensor& tin = net->tensors[in_tensor];
    const Tensor& to = net->tensors[out_tensor];
    const int span = dilation * (kernel - 1) + 1;
    const int ho = (tin.h + 2 * pad - span) / stride + 1, wo = (tin.w + 2 * pad - span) / stride + 1;
    const int C = pad8(channels);
    PIFPAF_CHECK_ARG(to.h == ho && to.w == wo, "dwconv output tensor shape mismatch");
    PIFPAF_CHECK_ARG(in_col_off % 8 == 0 && out_col_off % 8 == 0 && in_col_off + C <= tin.c && out_col_off + C <= to.c,
                     "dwconv column windows");
    PIFPAF_CUDA_TRY(cudaSetDevice(net->device));
    Op op; op.kind = OP_DW;
    float *d_w = nullptr, *d_b = nullptr;
    int rc = upload_dw_weights(net, weight, bias, channels, C, kernel * kernel, &d_w, &d_b);
    if (rc != PIFPAF_OK) return rc;
    DwArgs& a = op.dw;
    a.in = tin.data; a.ld_in = tin.c; a.in_col_off = in_col_off;
    a.out = to.data; a.ld_out = to.c; a.out_col_off = out_col_off;
    a.weight = d_w; a.bias = d_b;
    a.Hin = tin.h; a.Win = tin.w; a.Hout = ho; a.Wout = wo; a.C8 = C / 8;
    a.kernel = kernel; a.stride = stride; a.pad = pad; a.relu = relu;
    op.dw_dil = dilation;
    op.flops_per_image = 2.0 * ho * wo * channels * (double)kernel * kernel;
    op.bytes_per_image = ((double)tin.h * tin.w + (double)ho * wo) * channels * 2.0;
    choose_dw_kernels(net, op);
    if (op.dw_tma) {
        rc = make_tmap_dw(&op.tmap_dw, tin.data + in_col_off, (uint64_t)C, (uint64_t)tin.w, (uint64_t)tin.h,
                          (uint64_t)net->max_batch, (uint64_t)tin.c, op.dw_tma->box_w, op.dw_tma->box_h);
        if (rc != PIFPAF_OK) return rc;
    }
    op.touches = {in_tensor, out_tensor};
    op.dw_out_bytes_per_image = (double)ho * wo * channels * 2.0;
    net->ops.push_back(op);
    return PIFPAF_OK;
}

int pifpaf_net_maxpool(pifpaf_net_t* net, int32_t in_tensor, int32_t in_col_off, int32_t channels, int32_t stride,
                       int32_t out_tensor, int32_t out_col_off) {
    PIFPAF_CHECK_ARG(net != nullptr, "null argument");
    const int nt = (int)net->tensors.size();
    PIFPAF_CHECK_ARG(in_tensor >= 0 && in_tensor < nt && out_tensor >= 0 && out_tensor < nt, "bad tensor id");
    PIFPAF_CHECK_ARG(stride == 1 || stride == 2, "max pool stride must be 1 or 2");
    PIFPAF_CHECK_ARG(channels >= 1, "bad channel count");
    const Tensor& tin = net->tensors[in_tensor];
    const Tensor& to = net->tensors[out_tensor];
    const int ho = (tin.h - 1) / stride + 1, wo = (tin.w - 1) / stride + 1;     // (h + 2 * 1 - 3) / s + 1
    const int C = pad8(channels);
    PIFPAF_CHECK_ARG(to.h == ho && to.w == wo, "max pool output tensor shape mismatch");
    PIFPAF_CHECK_ARG(in_col_off % 8 == 0 && out_col_off % 8 == 0 && in_col_off + C <= tin.c && out_col_off + C <= to.c,
                     "max pool column windows");
    Op op; op.kind = OP_MAXPOOL;
    DwArgs& a = op.dw;
    a.in = tin.data; a.ld_in = tin.c; a.in_col_off = in_col_off;
    a.out = to.data; a.ld_out = to.c; a.out_col_off = out_col_off;
    a.Hin = tin.h; a.Win = tin.w; a.Hout = ho; a.Wout = wo; a.C8 = C / 8;
    a.kernel = 3; a.stride = stride; a.pad = 1; a.relu = 0;
    op.flops_per_image = 0;
    op.bytes_per_image = ((double)tin.h * tin.w + (double)ho * wo) * channels * 2.0;
    op.touches = {in_tensor, out_tensor};
    net->ops.push_back(op);
    return PIFPAF_OK;
}

int pifpaf_net_dw_conv1x1_scatter(pifpaf_net_t* net, int32_t in_tensor, int32_t in_col_off, int32_t channels,
                                  int32_t kernel, int32_t stride, int32_t pad,
                                  const float* dw_weight, const float* dw_bias, int32_t dw_relu,
                                  int32_t n_out, const float* weight, const float* bias, int32_t relu,
                                  int32_t n_pieces, const int32_t* piece_col0, const int32_t* piece_count,
                                  const int32_t* piece_tensor, const int32_t* piece_tensor_col) {
    PIFPAF_CHECK_ARG(net != nullptr && dw_weight != nullptr && weight != nullptr && piece_col0 && piece_count &&
                     piece_tensor && piece_tensor_col, "null argument");
    const int nt = (int)net->tensors.size();
    PIFPAF_CHECK_ARG(in_tensor >= 0 && in_tensor < nt, "bad tensor id");
    PIFPAF_CHECK_ARG(kernel == 5 && stride == 1 && pad == 2, "the fused depthwise -> 1x1 op covers 5x5, stride 1, pad 2");
    PIFPAF_CHECK_ARG(dw_relu >= ACT_NONE && dw_relu <= ACT_RELU && relu >= ACT_NONE && relu <= ACT_RELU,
                     "the fused depthwise -> 1x1 op takes activation codes 0 (none) and 1 (ReLU)");
    PIFPAF_CHECK_ARG(n_out >= 16 && n_out % 16 == 0 && n_out <= 512 && n_pieces >= 1, "n_out: multiple of 16, at most 512");
    const Tensor& tin = net->tensors[in_tensor];
    const int C = pad8(channels);
    PIFPAF_CHECK_ARG(in_col_off % 8 == 0 && in_col_off + C <= tin.c, "depthwise column window");
    PIFPAF_CUDA_TRY(cudaSetDevice(net->device));
    Op op; op.kind = OP_FUSED;
    float *d_dww = nullptr, *d_dwb = nullptr;
    int rc = upload_dw_weights(net, dw_weight, dw_bias, channels, C, 25, &d_dww, &d_dwb);
    if (rc != PIFPAF_OK) return rc;
    FusedArgs& f = op.fu;
    // column blocks of at most FD_MAX_BLOCK_N: one CTA (and one depthwise pass) per block
    const int n_blocks = (n_out + FD_MAX_BLOCK_N - 1) / FD_MAX_BLOCK_N;
    const int block_n = pad16((n_out + n_blocks - 1) / n_blocks);
    const int n_pad = block_n * n_blocks;
    f.dw_weight = d_dww; f.dw_bias = d_dwb; f.C = C; f.dw_relu = dw_relu; f.pad = pad;
    // 1x1 weights [n_out][channels] -> bf16 [n_pad][C]
    GemmWeights gw;
    rc = upload_gemm_weights(net, weight, bias, n_out, channels, 1, C, n_pad, &gw);
    if (rc != PIFPAF_OK) return rc;
    std::vector<int> map_tensor;      // k_dw_gemm has the per-lane scatter epilogue only: no store maps
    rc = upload_dest_groups(net, n_pad, n_out, tin.h, tin.w, n_pieces, piece_col0, piece_count, piece_tensor,
                            piece_tensor_col, &op.g.dest, &map_tensor);
    if (rc != PIFPAF_OK) return rc;

    GemmArgs& g = op.g;
    g.N = n_out; g.K = C; g.block_n = block_n; g.n_blocks = n_blocks;
    g.num_k_blocks = (C + BK - 1) / BK;
    g.bias = gw.bias; g.mode = MODE_SCATTER; g.relu = relu;
    g.conv_k = kernel; g.conv_stride = stride; g.conv_pad = pad; g.conv_dil = 1; g.conv_cblocks = g.num_k_blocks;
    g.Hi = tin.h; g.Wi = tin.w; g.Ho = tin.h; g.Wo = tin.w;
    g.tiles_x = (g.Wo + PW - 1) / PW; g.tiles_y = (g.Ho + PH - 1) / PH;
    op.a_tensor = in_tensor; op.rows_per_image = g.Ho * g.Wo; op.tiles_per_image = g.tiles_x * g.tiles_y;
    // ring depths: as deep as the shared memory allows, windows first (their TMA has the longest latency)
    const int cand[][2] = {{3, 2}, {2, 2}, {2, 1}, {1, 1}};
    bool fits = false;
    for (const auto& c : cand) {
        if (fused_smem_bytes(c[0], c[1], block_n, n_pad, C) <= GEMM_SMEM_BUDGET) {
            f.ws = c[0]; f.bs = c[1]; fits = true; break;
        }
    }
    PIFPAF_CHECK_ARG(fits, "fused depthwise -> 1x1 op does not fit in shared memory");
    op.smem = fused_smem_bytes(f.ws, f.bs, block_n, n_pad, C);
    op.n_real = gw.n_real;
    op.flops_per_image = 2.0 * (double)op.rows_per_image * ((double)gw.nnz + 25.0 * channels);
    op.bytes_per_image = (double)op.rows_per_image * (channels + gw.n_real) * 2.0;     // dw input once + 1x1 output once
    op.weight_bytes = (double)gw.nnz * 2.0 + 25.0 * channels * 4.0;
    using T = DwTile<1, PH, PW, 4, 1>;
    rc = make_tmap_dw(&op.tmap_dw, tin.data + in_col_off, (uint64_t)C, (uint64_t)tin.w, (uint64_t)tin.h,
                      (uint64_t)net->max_batch, (uint64_t)tin.c, T::IW, T::IH);
    if (rc != PIFPAF_OK) return rc;
    rc = make_tmap(&op.tmap_b, gw.w, (uint64_t)n_pad, (uint64_t)C, (uint64_t)C, (uint32_t)block_n);
    if (rc != PIFPAF_OK) return rc;
    op.touches.assign(piece_tensor, piece_tensor + n_pieces);
    op.touches.push_back(in_tensor);
    net->ops.push_back(op);
    return PIFPAF_OK;
}

int pifpaf_net_heads(pifpaf_net_t* net, int32_t in_tensor, int32_t k_cols, int32_t n_heads,
                     const int32_t* n_fields, const int32_t* n_comp, const int32_t* comp_ops,
                     const float* weight, const float* bias) {
    return pifpaf_net_heads_upsampled(net, in_tensor, k_cols, n_heads, n_fields, n_comp, comp_ops, 1, weight, bias);
}

int pifpaf_net_heads_upsampled(pifpaf_net_t* net, int32_t in_tensor, int32_t k_cols, int32_t n_heads,
                               const int32_t* n_fields, const int32_t* n_comp, const int32_t* comp_ops,
                               int32_t upsample_stride, const float* weight, const float* bias) {
    PIFPAF_CHECK_ARG(net != nullptr && weight != nullptr && n_fields && n_comp && comp_ops, "null argument");
    PIFPAF_CHECK_ARG(n_heads >= 1 && n_heads <= 4, "1..4 heads supported");
    PIFPAF_CHECK_ARG(upsample_stride >= 1 && upsample_stride <= 8, "upsample_stride must be in [1, 8]");
    PIFPAF_CHECK_ARG(in_tensor >= 0 && in_tensor < (int)net->tensors.size(), "bad tensor id");
    PIFPAF_CUDA_TRY(cudaSetDevice(net->device));
    const Tensor& tin = net->tensors[in_tensor];
    const int up = upsample_stride, up2 = up * up;
    // heads.py:336-343: low_cut = (up - 1) / 2, high_cut = ceil((up - 1) / 2)
    const int low = (up - 1) / 2, high = up / 2;
    const int out_h = tin.h * up - low - high, out_w = tin.w * up - low - high;
    PIFPAF_CHECK_ARG(out_h >= 1 && out_w >= 1, "feature map too small for this upsample_stride");
    int n_total = 0;
    for (int i = 0; i < n_heads; i++) n_total += n_fields[i] * n_comp[i] * up2;
    Op op; op.kind = OP_GEMM;
    int rc = emit_gemm(net, op, in_tensor, 0, k_cols, n_total, weight, bias);
    if (rc != PIFPAF_OK) return rc;
    GemmArgs& g = op.g;
    g.mode = MODE_HEADS; g.relu = 0;
    op.bytes_per_image += (double)out_h * out_w * (op.n_real / up2) * 4.0;
    std::vector<HeadCol> cols((size_t)g.block_n * g.n_blocks, HeadCol{0, 0, 0, 0});
    int col = 0, op_off = 0;
    for (int i = 0; i < n_heads; i++) {
        for (int f = 0; f < n_fields[i]; f++)
            for (int c = 0; c < n_comp[i]; c++)
                for (int dy = 0; dy < up; dy++)
                    for (int dx = 0; dx < up; dx++)
                        cols[col++] = HeadCol{i, f * n_comp[i] + c, comp_ops[op_off + c], (dy << 8) | dx};
        op_off += n_comp[i];
        net->head_fields[i] = n_fields[i]; net->head_comp[i] = n_comp[i];
        net->head_elems[i] = (size_t)net->max_batch * n_fields[i] * n_comp[i] * out_h * out_w;
        rc = net_alloc(net, &net->head_out[0][i], net->head_elems[i], true);
        if (rc != PIFPAF_OK) return rc;
        g.head_base[i] = net->head_out[0][i];
        g.head_planes[i] = n_fields[i] * n_comp[i];
    }
    HeadCol* d_cols = nullptr;
    rc = net_upload(net, &d_cols, cols); if (rc != PIFPAF_OK) return rc;
    g.head_cols = d_cols;
    g.hw = tin.h * tin.w; g.w = tin.w;
    g.up = up; g.up_low = low; g.out_h = out_h; g.out_w = out_w;
    plan_gemm_smem(op);
    net->n_heads = n_heads; net->head_h = out_h; net->head_w = out_w;
    op.touches = {in_tensor};
    net->ops.push_back(op);
    return PIFPAF_OK;
}

int pifpaf_net_head_output(pifpaf_net_t* net, int32_t head, float** dev_ptr,
                           int32_t* n_fields, int32_t* n_comp, int32_t* h, int32_t* w) {
    PIFPAF_CHECK_ARG(net != nullptr && head >= 0 && head < net->n_heads, "bad head index");
    if (dev_ptr) *dev_ptr = net->head_out[net->head_cur][head];     // the set the last forward wrote
    if (n_fields) *n_fields = net->head_fields[head];
    if (n_comp) *n_comp = net->head_comp[head];
    if (h) *h = net->head_h;
    if (w) *w = net->head_w;
    return PIFPAF_OK;
}

static int net_forward_impl(pifpaf_net_t* net, const float* images_dev, int32_t batch, int32_t gemm_impl,
                            cudaStream_t st, cudaEvent_t* events, const RawImages* u8 = nullptr) {
    PIFPAF_CHECK_ARG(net != nullptr, "null argument");
    PIFPAF_CHECK_ARG(images_dev != nullptr || u8 != nullptr || net->in_h == 0, "images pointer is null");
    PIFPAF_CHECK_ARG(batch >= 1 && batch <= net->max_batch, "batch exceeds max_batch");
    PIFPAF_CUDA_TRY(cudaSetDevice(net->device));
    if (!net->setup_synced) {
        // tensors were zero-filled and weights uploaded on the legacy default stream at emit time; `st` may be a
        // non-blocking stream that does not order itself behind it
        PIFPAF_CUDA_TRY(cudaDeviceSynchronize());
        net->setup_synced = true;
    }
    if (net->head_buffers == 2) net->head_cur ^= 1;
    if (net->pw_dw_planned != net->ops.size()) {
        const int rc = plan_pw_dw(net);
        if (rc != PIFPAF_OK) return rc;
    }
    int op_index = 0;
    net->elided_batch = 0;
    // PDL between consecutive ops (not in the per-op timing pass: the events would sit between the launches; not for
    // the first op: its predecessor in the stream is a copy or another forward's decode, not one of these kernels)
    const bool pdl_on = net->pdl && events == nullptr && gemm_impl == 0;
    for (Op& op : net->ops) {
        if (events) PIFPAF_CUDA_TRY(cudaEventRecord(events[op_index], st));
        const bool pdl = pdl_on && op_index > 0;
        op_index++;
        if (op.elided && gemm_impl == 0) {          // computed inside the fused launch of the next op (plan_pw_dw)
            net->elided_batch = batch;
            continue;
        }
        const int rc = launch_op(net, op, batch, gemm_impl, pdl, st, images_dev, u8);
        if (rc != PIFPAF_OK) return rc;
    }
    if (events) PIFPAF_CUDA_TRY(cudaEventRecord(events[op_index], st));
    return PIFPAF_OK;
}

int pifpaf_net_forward(pifpaf_net_t* net, const float* images_dev, int32_t batch, int32_t gemm_impl,
                       void* stream_v) {
    return net_forward_impl(net, images_dev, batch, gemm_impl, reinterpret_cast<cudaStream_t>(stream_v), nullptr);
}

int pifpaf_net_forward_u8(pifpaf_net_t* net, const uint8_t* images_nhwc_dev, int32_t batch, const float* mean,
                          const float* stdev, int32_t gemm_impl, void* stream_v) {
    PIFPAF_CHECK_ARG(images_nhwc_dev != nullptr && mean != nullptr && stdev != nullptr, "null argument");
    RawImages raw;
    raw.images = images_nhwc_dev;
    for (int c = 0; c < 3; c++) {
        PIFPAF_CHECK_ARG(stdev[c] > 0.f, "std must be positive");
        raw.mean[c] = mean[c]; raw.stdev[c] = stdev[c];
    }
    return net_forward_impl(net, nullptr, batch, gemm_impl, reinterpret_cast<cudaStream_t>(stream_v), nullptr, &raw);
}

int pifpaf_net_forward_timed(pifpaf_net_t* net, const float* images_dev, int32_t batch, int32_t gemm_impl,
                             void* stream_v, float* op_ms, int32_t* op_kind, double* op_flops, double* op_bytes) {
    PIFPAF_CHECK_ARG(net != nullptr && op_ms != nullptr, "null argument");
    PIFPAF_CUDA_TRY(cudaSetDevice(net->device));
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_v);
    const size_t n = net->ops.size();
    std::vector<cudaEvent_t> ev(n + 1);
    for (auto& e : ev) PIFPAF_CUDA_TRY(cudaEventCreate(&e));
    int rc = net_forward_impl(net, images_dev, batch, gemm_impl, st, ev.data());
    if (rc == PIFPAF_OK) {
        cudaError_t e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) { pifpaf::set_error("forward failed: %s", cudaGetErrorString(e)); rc = PIFPAF_E_CUDA; }
    }
    for (size_t i = 0; i < n && rc == PIFPAF_OK; i++) {
        cudaEventElapsedTime(&op_ms[i], ev[i], ev[i + 1]);
        const Op& op = net->ops[i];
        // the 1x1 -> depthwise pair that net_forward_impl skips and launch_dw runs as k_pw_dw
        const bool fused = gemm_impl == 0 && (op.elided || op.pw_dw);
        if (op_kind) op_kind[i] = fused ? OP_FUSED : op.kind;
        // an elided GEMM launches nothing (its events bracket no work) and its work is counted in the fused launch
        if (op_flops) op_flops[i] = !fused ? op.flops_per_image * batch : op.pw_dw ? op.pw_flops_per_image * batch : 0.0;
        if (op_bytes)
            op_bytes[i] = !fused ? op.bytes_per_image * batch + op.weight_bytes
                                 : op.pw_dw ? op.pw_bytes_per_image * batch + op.pw_weight_bytes : 0.0;
    }
    for (auto& e : ev) cudaEventDestroy(e);
    return rc;
}

int pifpaf_net_tap_tensor(pifpaf_net_t* net, int32_t id, int32_t batch, float* out, int64_t out_elems) {
    PIFPAF_CHECK_ARG(net != nullptr && id >= 0 && id < (int)net->tensors.size(), "bad tensor id");
    const Tensor& t = net->tensors[id];
    const long long n = (long long)batch * t.h * t.w * t.c;
    PIFPAF_CHECK_ARG(out != nullptr && out_elems >= n && batch <= net->max_batch, "output buffer too small");
    PIFPAF_CUDA_TRY(cudaSetDevice(net->device));
    // a tensor the last forward elided (the 1x1 output inside k_pw_dw): its GEMM runs now, at that forward's batch.
    // Its input (the stem output) is not overwritten within a forward, so this is what the two-kernel schedule wrote.
    if (net->elided_batch > 0)
        for (Op& op : net->ops)
            if (op.elided && op.g.out == t.data) {
                const int rc = launch_gemm(net, op, net->elided_batch, 0, false, 0);
                if (rc != PIFPAF_OK) return rc;
            }
    float* d_tmp = nullptr;
    PIFPAF_CUDA_TRY(cudaMalloc(reinterpret_cast<void**>(&d_tmp), sizeof(float) * n));
    const int rc = launch_k(false, k_bf16_to_f32, dim3(1024), dim3(256), 0, 0, t.data, d_tmp, n);
    const cudaError_t e = rc == PIFPAF_OK ? cudaMemcpy(out, d_tmp, sizeof(float) * n, cudaMemcpyDeviceToHost) : cudaSuccess;
    cudaFree(d_tmp);
    if (e != cudaSuccess) { pifpaf::set_error("tap copy failed: %s", cudaGetErrorString(e)); return PIFPAF_E_CUDA; }
    return rc;
}

int pifpaf_net_set_tensor(pifpaf_net_t* net, int32_t id, int32_t batch, const float* data, int64_t n_elems) {
    PIFPAF_CHECK_ARG(net != nullptr && id >= 0 && id < (int)net->tensors.size(), "bad tensor id");
    const Tensor& t = net->tensors[id];
    const long long n = (long long)batch * t.h * t.w * t.c;
    PIFPAF_CHECK_ARG(data != nullptr && n_elems == n && batch <= net->max_batch, "input size mismatch");
    PIFPAF_CUDA_TRY(cudaSetDevice(net->device));
    float* d_tmp = nullptr;
    PIFPAF_CUDA_TRY(cudaMalloc(reinterpret_cast<void**>(&d_tmp), sizeof(float) * n));
    int rc = PIFPAF_OK;
    cudaError_t e = cudaMemcpy(d_tmp, data, sizeof(float) * n, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) {
        rc = launch_k(false, k_f32_to_bf16, dim3(1024), dim3(256), 0, 0, d_tmp, t.data, n);
        if (rc == PIFPAF_OK) e = cudaDeviceSynchronize();
    }
    cudaFree(d_tmp);
    if (rc != PIFPAF_OK) return rc;
    if (e != cudaSuccess) { pifpaf::set_error("set_tensor failed: %s", cudaGetErrorString(e)); return PIFPAF_E_CUDA; }
    return PIFPAF_OK;
}

int pifpaf_net_set_head_buffers(pifpaf_net_t* net, int32_t n_buffers) {
    PIFPAF_CHECK_ARG(net != nullptr && (n_buffers == 1 || n_buffers == 2), "n_buffers must be 1 or 2");
    PIFPAF_CUDA_TRY(cudaSetDevice(net->device));
    if (n_buffers == 2) {
        for (int i = 0; i < net->n_heads; i++) {
            if (net->head_out[1][i] != nullptr) continue;
            int rc = net_alloc(net, &net->head_out[1][i], net->head_elems[i], true);
            if (rc != PIFPAF_OK) return rc;
        }
        net->setup_synced = false;
    } else {
        net->head_cur = 0;
    }
    net->head_buffers = n_buffers;
    return PIFPAF_OK;
}

int pifpaf_net_set_sm_limit(pifpaf_net_t* net, int32_t n_sm) {
    PIFPAF_CHECK_ARG(net != nullptr && n_sm >= 0, "bad argument");
    net->sm_limit = n_sm;
    return PIFPAF_OK;
}

double pifpaf_net_flops_per_image(pifpaf_net_t* net) {
    if (!net) return 0.0;
    double f = 0.0;
    for (const Op& op : net->ops) f += op.flops_per_image;
    return f;
}

int32_t pifpaf_net_num_ops(pifpaf_net_t* net) { return net ? (int32_t)net->ops.size() : 0; }

}  // extern "C"
