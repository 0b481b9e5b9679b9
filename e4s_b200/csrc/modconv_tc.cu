// Tensor-core 3x3 convolutions of the library (sm_90a): the region-selected modulated convolution (plain and up-sampling
// layers; an up-sampling layer is a transposed-convolution GEMM followed by a streaming blur pass - over (pixel, region)
// rows when masked - or four output-parity convolutions on the input grid), the encoder's plain convolution, and the
// input / style gradient of the modulated one.
//
// The convolution kernels share the split-precision MMA step (split_mma, SplitAcc), the work-item decode (decode_item)
// and the layer epilogue (epilogue2; epilogue4 in the blur passes).
//
// Plain modulated layers and (DENSE mode) the plain convolutions of ESRGAN's RRDBNet run on conv3x3_rs_kernel (below):
// fp32 halo tiles in shared memory, the A operand built in registers; the unmasked transposed-convolution GEMM on its
// transposed-convolution mode (CONVT), the masked one on its gathered-row mode (ROWS).  Everything else - the folded
// parity kernels, the encoder convolution and the gradient - runs on conv3x3_wgmma_kernel, described here.  A work item is an 8 x 16 pixel tile
// (M = 128 rows) times an N tile of 32 or 64 output channels (one output parity of an up-sampling layer, or all four in
// turn); K runs over (parity plane, tap, 32-channel chunk).  Per K step the 256 threads stage
//   A: the 128 x 32 operand tile read from global memory at the tap's offset and scaled while staging - by the style of
//      each row's own output pixel (forward: every row may belong to another region, so a tile mixing regions needs no
//      extra pass), or by act'(y) * demod of the region whose pass it is (gradient: rows of other regions are zero);
//   B: the N x 32 weight tile from the pre-split bf16 planes,
// both as bf16 hi / lo planes (x = hi + lo to ~2^-17) in the no-swizzle K-major core-matrix layout of wgmma.  The two
// warpgroups (64 rows each) issue asynchronous wgmma.mma_async m64nNk16 with both operands from shared memory into
// fp32 register accumulators (split_mma).  The operand tiles go through a four-stage shared-memory ring: while the MMAs
// of step k run, the threads store step k + 2 (loaded from global memory one step earlier) and issue the loads of step
// k + 3; one barrier per K step.  The operands cannot be copied by TMA: every element is scaled and split on its way
// into shared memory.  Every output element is accumulated in a fixed order, so the forward is bit reproducible; the
// gradient sums split work items and style gradients with atomics.
#include <cuda_bf16.h>
#include <cstdio>
#include <cstdlib>
#include <initializer_list>
#include <type_traits>

#include "common.cuh"

namespace wgmma_conv {

constexpr int TH = 8, TW = 16, M = TH * TW;     // pixel tile: 8 rows x 16 columns
constexpr int KC = 32;                          // channels per K step
constexpr int NUM_THREADS = 256;                // two warpgroups, 64 pixel rows each
constexpr int NSTAGE = 4;                       // operand ring: step k in flight, k + 1 ready, k + 2 being stored
// No-swizzle K-major core-matrix layout (8 rows x 16 bytes per core matrix): element (r, k) of a 32-channel tile at byte
// (r / 8) * SBO + (k / 8) * LBO + (r % 8) * 16 + (k % 8) * 2.
constexpr int LBO = 128, SBO = 512;
constexpr int A_PLANE = M * KC * 2;             // 8 KB per bf16 plane
constexpr float SQRT2 = 1.41421356237309515f;
// A row of the masked transposed-convolution GEMM: T' pixel (m, n) computed with the style of region r, packed as
// m (14 bits) | n (13 bits) | r (5 bits).
constexpr int ROW_NBITS = 13;
__host__ __device__ constexpr uint32_t row_pack(int m, int n, int r) {
    return ((uint32_t)m << (ROW_NBITS + 5)) | ((uint32_t)n << 5) | (uint32_t)r;
}

// FWD_RS: launch conv3x3_rs_kernel (host side only).
// FWD_BIAS: FWD with the epilogue relu?(acc + bias + residual) (epilogue_bias2) in place of epilogue2.
// FWD_DENSE: launch conv3x3_rs_kernel in its plain mode (host side only): unscaled pitched operands, the ESRGAN epilogue.
// FWD_REFL: FWD_DENSE with reflection padding in the halo copy (Params::reflect) in place of the zero fill.
// FWD_PW: FWD_DENSE as a 1x1 (pointwise) convolution: no halo, several K chunks per ring slot (Params::in_stride, r_up).
// FWD_VOL: FWD_DENSE as a 3x3x3 convolution over a mosaic of depth slices (VolGrid).
// FWD_SPADE: FWD_DENSE whose output columns are interleaved (gamma, beta) pairs of a SPADE modulation, applied in the
// epilogue to the instance-normalised input (Params::norm_x); neither the normalised input nor gamma / beta is written.
// FWD_PWF: FWD_PW with the result multiplied by a per-pixel factor (Params::factor).
enum Mode { FWD = 0, BWD = 2, FWD_RS = 3, FWD_BIAS = 4, FWD_DENSE = 5, FWD_REFL = 6, FWD_PW = 7, FWD_VOL = 8,
            FWD_SPADE = 9, FWD_PWF = 10 };
// conv3x3_rs_kernel's epilogue variants (the existing modes: EPI_PLAIN)
enum Epilogue { EPI_PLAIN = 0, EPI_FACTOR = 1, EPI_SPADE = 2 };

// FWD_VOL: the 3x3x3 convolution (padding 1) over [B, H, W, D, C] tensors as a 3x3 convolution over a mosaic of its
// B * D depth slices ("cells", b-major), each H x W (the output grid).  Cell i sits at cell row i / ncx, column i % ncx;
// with gutter 1 the cells are (H + 1) x (W + 1) apart, so the zero gutter row and column between them are the in-plane
// padding and small slices share pixel tiles; with gutter 0 (H a multiple of the tile height, ncx = 1) the slices are
// stacked and no tile straddles two of them.  K is (kz, Cin): chunk kc reads depth z + kc / (Cin / 32) - 1 of the
// pixel's cell, zero outside [0, D).  Voxel (y, x, z) of the input starts at float (y W + x) a_ld + z vox_in, of the output
// at (y W + x) out_ld + z vox_out (a_ld = D vox_in, out_ld = D vox_out): a channel slice of a wider [B, H, W, D, C'] buffer
// when the voxel pitch exceeds the channel count (the hourglass concatenations of face-vid2vid's dense-motion network).
struct VolGrid {
    int depth, ncx, cells, gutter;
};

// Params p{}: every member without a default below starts zero / NULL.
struct Params {
    const float* a;          // FWD: x [B, H, W, Cin]; BWD: gy [B, Ho, Wo, Cout]
    const float* y;          // BWD: forward output (activation derivative) or NULL
    const float* x;          // BWD: forward input (style gradient) or NULL
    const __nv_bfloat16* wt; // weight planes (see the entry points)
    const float* s;          // [B, ncls, Cin] styles (encoder: per-sample scale [B, Cin]; FWD_SPADE: [B, C]) or NULL
    const float* shift;      // encoder: [B, Cin] added to in-image pixels (FWD_SPADE: [B, C]), or NULL
    const float* demod;      // [B, ncls, Cout] or NULL
    const uint8_t* label;    // [B, Ho, Wo] or NULL
    const float* noise;
    const float* noise_w;
    const float* bias;
    const float* slope;      // act == 2: PReLU slopes [Cout]
    float* out;              // FWD: y; BWD: gx [B, H, W, Cin] (may be NULL)
    float* gs;               // BWD: [B, ncls, Cin] accumulated, or NULL
    int batch, h, w, kch, nch;   // kch: channels along K (FWD Cin, BWD Cout); nch: along N (FWD Cout, BWD Cin)
    int ncls, noise_b = 1, act, up, out_stride = 1;    // noise_b: noise batch, 1 or batch
    int ntaps;
    int taps[16];            // K taps (row-major 3x3 index)
    VolGrid vol;             // FWD_VOL: the mosaic of depth slices
    int mh, mw;              // output row grid (FWD: the input grid, or one pixel larger for the transposed convolution)
    int tiles_x, tiles_y, n_tiles, gsplit = 1, hsplit = 1, atomic_gx;
    // N tiles per work item of conv3x3_wgmma_kernel: always 1.  The gradient still loops over them: without that loop
    // nvcc schedules it differently, and its 64-channel instantiation ran ~5 % slower (H100 80GB HBM3, 400 W).
    int n_sub = 1;
    int parity_items;        // up-sampling forward: 1 = one output parity per work item, 0 = all four in one item
    // masked transposed-convolution GEMM: row_count [B] rows in each sample's list, cap rows reserved per sample.
    // conv3x3_rs_kernel's ROWS mode: row i of sample b is the packed (m, n, region) rows[b * cap + i], out is [B, cap, nch];
    // samples with row_count > cap are skipped.  FWD with row_count: the folded fallback - only samples with
    // row_count > cap are computed.
    // FWD_PWF: the per-pixel factor [B, mh, mw] (shares the storage of rows, which the pointwise mode never reads)
    union { const uint32_t* rows; const float* factor; };
    const int* row_count;
    union { int cap; int rup_ld; int vox_out; int norm_ld; };     // FWD_PW: rup_ld; FWD_VOL: vox_out (see VolGrid)
    // FWD_BIAS: added before the activation, laid out like out (read at the offset of the stored element), or NULL
    const float* residual;
    // FWD_DENSE: pixel pitches of a and out (floats, multiples of 4); the epilogue t = (acc + bias) * alpha, t += residual,
    // t = t * beta + residual2 (each residual optional, pitched like out), then leaky ReLU with slope lrelu (1: none).
    // up: the halo is read from the half-size input at (sy >> 1, sx >> 1) (nearest 2x up-sampling; h, w: the output grid).
    int a_ld, out_ld;
    // FWD_PW: residual_up; FWD_SPADE: norm_x, the input x of the normalisation, pixel pitch norm_ld, at the output grid
    // (norm_half 0) or at half of it, read at (y >> 1, x >> 1) (norm_half 1)
    union { const float* residual2; const float* residual_up; const float* norm_x; };
    float alpha, beta, lrelu;
    // FWD_REFL: halo pixel (sy, sx) outside the grid reads, per axis, 1: the mirror pixel (-1 -> 1, h -> h - 2: reflection
    // padding 1); 2: the nearest edge pixel (replicate).  Reflection padding of the nearest-2x up-sampled grid is replicate
    // padding at the source (and so at the up-sampled grid: the halo copy then halves the index); for a stride-2 convolution
    // over the space-to-depth operand (taps {-1, 0}^2) reflection padding 1 is row and column -1 replicating row and column 0.
    // FWD_PW (shares the storage of members its kernels never read, so that Params keeps its size and layout): output pixel
    // (y, x) reads input pixel (in_stride y, in_stride x) (h, w: the input grid; mh, mw: the output grid); ntaps = K chunks
    // per ring slot (taps[i] = i); after the activation, residual_up [B, mh / 2, mw / 2] (pixel pitch rup_ld) is added at
    // (y >> 1, x >> 1), or nothing when NULL.
    union { int reflect; int in_stride; int vox_in; int norm_half; };
};

// Shared-memory matrix descriptor: start address, LBO, SBO (16-byte units), no swizzle.
__device__ __forceinline__ uint64_t sdesc(uint32_t saddr) {
    return (uint64_t)((saddr & 0x3FFFF) >> 4) | ((uint64_t)(LBO >> 4) << 16) | ((uint64_t)(SBO >> 4) << 32);
}
// m64 x N x k16, N = 2 * NR: A from shared memory at address sa (N = 32, 64) or from registers (N = 32, 64, 128), B from
// shared memory at address sb;
// accumulate = 0: D = A B (the first MMA of an accumulation), else D += A B
template <int NR>
__device__ __forceinline__ void wgmma(float (&d)[NR], uint32_t sa, uint32_t sb, int accumulate) {
    const uint64_t da = sdesc(sa), db = sdesc(sb);
    if constexpr (NR == 32)
        asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
                     "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, 0, 0;\n}"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                     : "l"(da), "l"(db), "r"(accumulate));
    else
        asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
                     "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, 0, 0;\n}"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
                     : "l"(da), "l"(db), "r"(accumulate));
}
template <int NR>
__device__ __forceinline__ void wgmma(float (&d)[NR], const uint32_t (&a)[4], uint32_t sb, int accumulate) {
    const uint64_t db = sdesc(sb);
    if constexpr (NR == 64)
        asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %69, 0;\n"
                     "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, {%64,%65,%66,%67}, %68, p, 1, 1, 0;\n}"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(accumulate));
    else if constexpr (NR == 32)
        asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %37, 0;\n"
                     "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, {%32,%33,%34,%35}, %36, p, 1, 1, 0;\n}"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(accumulate));
    else
        asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %21, 0;\n"
                     "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, {%16,%17,%18,%19}, %20, p, 1, 1, 0;\n}"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across an asynchronous MMA
template <int NR>
__device__ __forceinline__ void fence_regs(float (&d)[NR]) {
#pragma unroll
    for (int i = 0; i < NR; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ uint32_t pack2(__nv_bfloat16 lo_elem, __nv_bfloat16 hi_elem) {
    return (uint32_t)__bfloat16_as_ushort(lo_elem) | ((uint32_t)__bfloat16_as_ushort(hi_elem) << 16);
}
// four fp32 values -> bf16 hi plane and residual lo plane, 8 bytes each
__device__ __forceinline__ void split_store4(float4 v, __nv_bfloat16* hi, __nv_bfloat16* lo) {
    const __nv_bfloat16 h0 = __float2bfloat16_rn(v.x), h1 = __float2bfloat16_rn(v.y), h2 = __float2bfloat16_rn(v.z),
                        h3 = __float2bfloat16_rn(v.w);
    const __nv_bfloat16 l0 = __float2bfloat16_rn(v.x - __bfloat162float(h0)), l1 = __float2bfloat16_rn(v.y - __bfloat162float(h1)),
                        l2 = __float2bfloat16_rn(v.z - __bfloat162float(h2)), l3 = __float2bfloat16_rn(v.w - __bfloat162float(h3));
    *reinterpret_cast<uint2*>(hi) = make_uint2(pack2(h0, h1), pack2(h2, h3));
    *reinterpret_cast<uint2*>(lo) = make_uint2(pack2(l0, l1), pack2(l2, l3));
}
__device__ __forceinline__ float4 ld4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ float4 mul4(float4 a, float4 b) { return make_float4(a.x * b.x, a.y * b.y, a.z * b.z, a.w * b.w); }
__device__ __forceinline__ float actd(float y) { return y > 0.f ? SQRT2 : 0.2f * SQRT2; }

// A warpgroup's fp32 accumulators of an m64 x NT tile in the split-precision scheme: x = x_hi + x_lo, w = w_hi + w_lo
// in bf16, d = x_lo w_hi + x_hi w_lo + x_hi w_hi (~1e-5 relative to fp32).  STK (N tiles of 32): the w_hi and w_lo
// planes of a stage are contiguous along N, so ONE MMA of width 2 NT multiplies x_hi by both and a second one of width
// NT adds x_lo w_hi: two MMA instructions per K16 slice instead of three (the small-N layers issue many short MMAs);
// fold() adds the halves after the K loop.  Register 4 j + 2 h + e of d: row 16 (warp % 4) + lane / 4 + 8 h of the
// warpgroup's 64, column 8 j + 2 (lane % 4) + e.
template <int NT>
struct SplitAcc {
    static constexpr bool STK = NT == 32;
    static constexpr int NR = NT / 2;             // registers per thread
    float s[STK ? 2 * NR : 1], l[STK ? NR : 1];   // STK: [x_hi w_hi | x_hi w_lo] and x_lo w_hi
    float d[NR];
    __device__ __forceinline__ void fence() {
        fence_regs(d);
        fence_regs(s);
        fence_regs(l);
    }
    __device__ __forceinline__ void fold() {
        if constexpr (STK) {
#pragma unroll
            for (int i = 0; i < NR; ++i) d[i] = s[i] + s[i + NR] + l[i];
        }
    }
};

// The MMAs of one K16 slice, x_hi / x_lo from shared memory or registers, w_hi / w_lo from shared memory; accumulate = 0
// starts the sum.  The product order fixes every output's sum order.
template <int NT, typename A>
__device__ __forceinline__ void split_mma(SplitAcc<NT>& acc, const A& a_hi, const A& a_lo, uint32_t b_hi, uint32_t b_lo,
                                          int accumulate) {
    if constexpr (SplitAcc<NT>::STK) {
        wgmma(acc.s, a_hi, b_hi, accumulate);     // N = 2 NT over the w_hi and w_lo rows
        wgmma(acc.l, a_lo, b_hi, accumulate);
    } else {
        wgmma(acc.d, a_lo, b_hi, accumulate);
        wgmma(acc.d, a_hi, b_lo, 1);
        wgmma(acc.d, a_hi, b_hi, 1);
    }
}

// The layer epilogue act(a * demod + (noise + bias)).  act 1: leaky ReLU scaled by sqrt(2); act 2: PReLU (the encoder's
// convolution; compiled where PRELU).  epilogue2 stores channels n, n + 1 of a pixel of region cls of sample b at dst + n.
template <bool PRELU>
__device__ __forceinline__ void epilogue2(const Params& p, int b, int cls, int n, float z, float a0, float a1, float* dst) {
    float2 d = make_float2(1.f, 1.f), bv = make_float2(0.f, 0.f);
    if (p.demod) d = __ldg(reinterpret_cast<const float2*>(p.demod + ((int64_t)b * p.ncls + cls) * p.nch + n));
    if (p.bias) bv = __ldg(reinterpret_cast<const float2*>(p.bias + n));
    float2 o = make_float2(a0 * d.x + (z + bv.x), a1 * d.y + (z + bv.y));
    if (p.act == 1) {
        o.x = lrelu_scaled(o.x, 0.2f, SQRT2);
        o.y = lrelu_scaled(o.y, 0.2f, SQRT2);
    } else if (PRELU && p.act == 2) {
        const float2 sl = __ldg(reinterpret_cast<const float2*>(p.slope + n));
        o.x = o.x > 0.f ? o.x : o.x * sl.x;
        o.y = o.y > 0.f ? o.y : o.y * sl.y;
    }
    *reinterpret_cast<float2*>(dst + n) = o;
}
// FWD_BIAS: o = acc + bias[n] + residual, then ReLU when p.act; res points at the residual element of dst (or NULL)
__device__ __forceinline__ void epilogue_bias2(const Params& p, int n, float a0, float a1, const float* res, float* dst) {
    float2 o = make_float2(a0, a1);
    if (p.bias) {
        const float2 bv = __ldg(reinterpret_cast<const float2*>(p.bias + n));
        o.x += bv.x, o.y += bv.y;
    }
    if (res) {
        const float2 rv = *reinterpret_cast<const float2*>(res + n);
        o.x += rv.x, o.y += rv.y;
    }
    if (p.act) o.x = fmaxf(o.x, 0.f), o.y = fmaxf(o.y, 0.f);
    *reinterpret_cast<float2*>(dst + n) = o;
}
// FWD_DENSE, in the order of ESRGAN's modules: x5 = acc + bias; x5 * alpha + r0 (residual dense block); (...) * beta + r1
// (RRDB); leaky ReLU.  ro: offset of dst from p.out, where the residuals are read (each element by the thread storing it)
__device__ __forceinline__ void epilogue_dense2(const Params& p, int n, float a0, float a1, int64_t ro, float* dst) {
    float2 o = make_float2(a0, a1);
    if (p.bias) {
        const float2 bv = __ldg(reinterpret_cast<const float2*>(p.bias + n));
        o.x += bv.x, o.y += bv.y;
    }
    o.x *= p.alpha, o.y *= p.alpha;
    if (p.residual) {
        const float2 rv = *reinterpret_cast<const float2*>(p.residual + ro + n);
        o.x += rv.x, o.y += rv.y;
    }
    if (p.residual2) {
        const float2 rv = *reinterpret_cast<const float2*>(p.residual2 + ro + n);
        o.x = o.x * p.beta + rv.x, o.y = o.y * p.beta + rv.y;
    }
    if (p.lrelu != 1.f) {
        o.x = o.x > 0.f ? o.x : o.x * p.lrelu;
        o.y = o.y > 0.f ? o.y : o.y * p.lrelu;
    }
    *reinterpret_cast<float2*>(dst + n) = o;
}
// FWD_PW: t = (acc + bias) * alpha; t += r0; leaky ReLU; t += up (FPN's lateral + nearest-up-sampled coarser level), in
// that order; FACTOR (FWD_PWF): then t *= f.  ro as epilogue_dense2; up: the residual_up pixel of this output pixel, or NULL
template <bool FACTOR = false>
__device__ __forceinline__ void epilogue_pw2(const Params& p, int n, float a0, float a1, int64_t ro, const float* up, float f,
                                             float* dst) {
    float2 o = make_float2(a0, a1);
    if (p.bias) {
        const float2 bv = __ldg(reinterpret_cast<const float2*>(p.bias + n));
        o.x += bv.x, o.y += bv.y;
    }
    o.x *= p.alpha, o.y *= p.alpha;
    if (p.residual) {
        const float2 rv = *reinterpret_cast<const float2*>(p.residual + ro + n);
        o.x += rv.x, o.y += rv.y;
    }
    if (p.lrelu != 1.f) {
        o.x = o.x > 0.f ? o.x : o.x * p.lrelu;
        o.y = o.y > 0.f ? o.y : o.y * p.lrelu;
    }
    if (up) {
        const float2 uv = *reinterpret_cast<const float2*>(up + n);
        o.x += uv.x, o.y += uv.y;
    }
    if constexpr (FACTOR) o.x *= f, o.y *= f;
    *reinterpret_cast<float2*>(dst + n) = o;
}
// FWD_SPADE: columns n, n + 1 are (gamma, beta) of channel c = n / 2; xn = x s + t (the instance norm of x, s and t per
// sample and channel), o = xn (1 + (gamma + b_gamma)) + (beta + b_beta), then leaky ReLU with slope lrelu (1: none).
// xp: the input pixel of x, dst: the output pixel
__device__ __forceinline__ void epilogue_spade(const Params& p, int b, int n, float a0, float a1, const float* xp, float* dst) {
    const int c = n >> 1;
    const int64_t sc = (int64_t)b * (p.nch >> 1) + c;
    const float2 bv = __ldg(reinterpret_cast<const float2*>(p.bias + n));
    const float xn = fmaf(__ldg(xp + c), __ldg(p.s + sc), __ldg(p.shift + sc));
    float o = xn * (1.f + (a0 + bv.x)) + (a1 + bv.y);
    if (p.lrelu != 1.f) o = o > 0.f ? o : o * p.lrelu;
    dst[c] = o;
}
__device__ __forceinline__ float4 epilogue4(float4 a, float4 d, float z, float4 bv, int act) {
    float4 o = make_float4(a.x * d.x + (z + bv.x), a.y * d.y + (z + bv.y), a.z * d.z + (z + bv.z), a.w * d.w + (z + bv.w));
    if (act) {
        o.x = lrelu_scaled(o.x, 0.2f, SQRT2);
        o.y = lrelu_scaled(o.y, 0.2f, SQRT2);
        o.z = lrelu_scaled(o.z, 0.2f, SQRT2);
        o.w = lrelu_scaled(o.w, 0.2f, SQRT2);
    }
    return o;
}

// region of the pixel at label[i]: labels past the last region count as the last one
__device__ __forceinline__ int region(const uint8_t* label, int ncls, int64_t i) { return min((int)label[i], ncls - 1); }

// Work item idx: pixel tile (tx, ty), sample b, first channel n0 of its N tile of nt channels (tx fastest), and with
// REST the index past the N tile (rest).
struct Item {
    int tx, ty, b, n0, rest;
};
template <bool REST>
__device__ __forceinline__ Item decode_item(const Params& p, int idx, int nt) {
    Item it;
    it.tx = idx % p.tiles_x;
    idx /= p.tiles_x;
    it.ty = idx % p.tiles_y;
    idx /= p.tiles_y;
    it.b = idx % p.batch;
    idx /= p.batch;
    it.n0 = (REST ? idx % p.n_tiles : idx) * nt;
    it.rest = REST ? idx / p.n_tiles : 0;
    return it;
}
template <int NT, int MODE>
__global__ void __launch_bounds__(NUM_THREADS, (MODE == BWD || NT == 32) ? 1 : 2) conv3x3_wgmma_kernel(const Params p) {
    constexpr bool GRAD = MODE == BWD;
    static_assert(NT == 32 || NT == 64, "N tiles of 32 or 64");
    constexpr int NR = NT / 2;                        // accumulator registers per thread (m64 x NT per warpgroup)
    constexpr int BVEC = NT * KC / 8;                 // 16-byte vectors per B plane and K step
    constexpr int BV = (BVEC + NUM_THREADS - 1) / NUM_THREADS;
    constexpr int B_PLANE = NT * KC * 2;
    constexpr int STAGE = 2 * A_PLANE + 2 * B_PLANE;  // [A hi | A lo | B hi | B lo]
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    __shared__ uint32_t s_classes;

    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const int wg = warp >> 2, wi = warp & 3;          // warpgroup (rows 64 wg ..), warp within it
    Item it = decode_item<true>(p, blockIdx.x, NT * p.n_sub);
    const int b = it.b, idx = it.rest;
    int n0 = it.n0;
    const int mul = p.up ? 2 : 1;
    const int H = p.h, W = p.w, MH = p.mh, MW = p.mw, Ho = MH * mul, Wo = MW * mul;
    const int y0 = it.ty * TH, x0 = it.tx * TW;
    if (!GRAD && p.row_count && __ldg(p.row_count + b) <= p.cap) return;    // masked fallback: overflowed samples only
    const int nphw = p.up ? 4 : 1;                    // parity planes of the weights
    // FWD: idx = output parity of the item.  BWD: idx = region-pass group + gsplit * parity-plane group.
    int par = GRAD ? 0 : idx;
    const int g = GRAD ? idx % p.gsplit : 0;
    const int ph0 = GRAD ? (idx / p.gsplit) * (nphw / p.hsplit) : 0;
    const int nph_k = GRAD ? nphw / p.hsplit : 1;
    int py = par >> 1, px = par & 1;
    const int c4 = t & 7, rr = t >> 3;                // A staging: channel group, first row
    const int nchunks = p.kch / KC;
    const int nsteps = nph_k * p.ntaps * nchunks;
    const int64_t plane = (int64_t)p.nch * p.kch;

    // forward: region of each staged row's own output pixel
    int rcls[4] = {0, 0, 0, 0};
    auto row_classes = [&]() {
        if (!p.label) return;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int r = rr + 32 * j, iy = y0 + (r >> 4), ix = x0 + (r & 15);
            if (iy < MH && ix < MW) rcls[j] = region(p.label, p.ncls, ((int64_t)b * Ho + iy * mul + py) * Wo + ix * mul + px);
        }
    };

    float4 av[4], am[4], ad;
    bool aok[4];
    uint4 bh[BV], bl[BV];
    auto load = [&](int step, int pass) {
        const int kc = step % nchunks;
        const int rest = step / nchunks;
        const int tap = p.taps[rest % p.ntaps];
        const int ph = ph0 + rest / p.ntaps;
        const int dy = tap / 3, dx = tap % 3;
        const int k = kc * KC + c4 * 4;
        if (GRAD) ad = p.demod ? ld4(p.demod + ((int64_t)b * p.ncls + pass) * p.kch + k) : make_float4(1.f, 1.f, 1.f, 1.f);
        else ad = p.shift ? ld4(p.shift + (int64_t)b * p.kch + k) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int r = rr + 32 * j;
            const int iy = y0 + (r >> 4), ix = x0 + (r & 15);
            const int sy = iy + dy - 1, sx = ix + dx - 1;
            bool ok = iy < MH && ix < MW && sy >= 0 && sy < H && sx >= 0 && sx < W;
            av[j] = make_float4(0.f, 0.f, 0.f, 0.f);
            am[j] = make_float4(1.f, 1.f, 1.f, 1.f);
            if (GRAD) {
                const int64_t gp = ((int64_t)b * Ho + sy * mul + (ph >> 1)) * Wo + sx * mul + (ph & 1);
                if (ok && p.label) ok = region(p.label, p.ncls, gp) == pass;
                if (ok) {
                    av[j] = ld4(p.a + gp * p.kch + k);
                    if (p.y) am[j] = ld4(p.y + gp * p.kch + k);
                }
            } else if (ok) {
                av[j] = ld4(p.a + (((int64_t)b * H + sy) * W + sx) * p.kch + k);
                if (p.s) am[j] = ld4(p.s + ((int64_t)b * p.ncls + rcls[j]) * p.kch + k);
            }
            aok[j] = ok;
        }
#pragma unroll
        for (int v = 0; v < BV; ++v) {                // B: 16-byte vectors of both planes
            const int e = t + NUM_THREADS * v;
            if (e < BVEC) {
                const int n = n0 + (e >> 2), kk = kc * KC + (e & 3) * 8;
                const int wph = GRAD ? ph : par;
                const int64_t off = (int64_t)(wph * 9 + tap) * plane + (int64_t)n * p.kch + kk;
                bh[v] = __ldg(reinterpret_cast<const uint4*>(p.wt + off));
                bl[v] = __ldg(reinterpret_cast<const uint4*>(p.wt + (int64_t)nphw * 9 * plane + off));
            }
        }
    };
    auto store = [&](int buf) {
        uint8_t* st = smem + buf * STAGE;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int r = rr + 32 * j;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (aok[j]) {
                if (GRAD) {
                    const float4 d = p.y ? make_float4(actd(am[j].x), actd(am[j].y), actd(am[j].z), actd(am[j].w)) : am[j];
                    v = mul4(mul4(av[j], d), ad);
                } else {
                    v = make_float4(av[j].x * am[j].x + ad.x, av[j].y * am[j].y + ad.y, av[j].z * am[j].z + ad.z,
                                    av[j].w * am[j].w + ad.w);
                }
            }
            const int off = (r >> 3) * SBO + (c4 >> 1) * LBO + (r & 7) * 16 + (c4 & 1) * 8;
            split_store4(v, reinterpret_cast<__nv_bfloat16*>(st + off), reinterpret_cast<__nv_bfloat16*>(st + A_PLANE + off));
        }
#pragma unroll
        for (int v = 0; v < BV; ++v) {
            const int e = t + NUM_THREADS * v;
            if (e < BVEC) {
                const int n = e >> 2;
                const int off = 2 * A_PLANE + (n >> 3) * SBO + (e & 3) * LBO + (n & 7) * 16;
                *reinterpret_cast<uint4*>(st + off) = bh[v];
                *reinterpret_cast<uint4*>(st + off + B_PLANE) = bl[v];
            }
        }
    };
    SplitAcc<NT> acc{};                               // zero: the fences read every register
    const uint32_t smem_s = (uint32_t)__cvta_generic_to_shared(smem);
    // the split-precision products of one K step, both K16 slices, on ring slot `buf`
    auto issue = [&](int buf, bool first) {
        const uint32_t a_hi = smem_s + buf * STAGE + wg * (64 / 8) * SBO, a_lo = a_hi + A_PLANE;
        const uint32_t b_hi = smem_s + buf * STAGE + 2 * A_PLANE, b_lo = b_hi + B_PLANE;
        acc.fence();
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < KC / 16; ++ks) {
            const uint32_t ko = ks * 2 * LBO;
            const int accumulate = (first && ks == 0) ? 0 : 1;
            split_mma(acc, a_hi + ko, a_lo + ko, b_hi + ko, b_lo + ko, accumulate);
        }
        wgmma_commit();
        acc.fence();
    };
    // Ring: slot k % NSTAGE holds step k.  Iteration k issues step k, waits until only it is in flight (so step k - 1 is
    // done in this warpgroup), stores step k + 2 into the slot of step k - 2 (done in both warpgroups: the barrier of
    // iteration k - 1 followed their waits), loads step k + 3 into registers, and meets the other threads at the barrier.
    // (the first MMA of a pass overwrites the accumulators: no register write may sit between asynchronous MMAs)
    auto run = [&](int pass) {
        load(0, pass);
        store(0);
        if (1 < nsteps) load(1, pass), store(1);
        if (2 < nsteps) load(2, pass);
        fence_proxy_async();
        __syncthreads();
#pragma unroll 1
        for (int st = 0; st < nsteps; ++st) {
            issue(st % NSTAGE, st == 0);
            wgmma_wait<1>();
            acc.fence();
            if (st + 2 < nsteps) store((st + 2) % NSTAGE);
            if (st + 3 < nsteps) load(st + 3, pass);
            fence_proxy_async();
            __syncthreads();
        }
        wgmma_wait<0>();
        acc.fence();
        __syncthreads();                              // every slot free before a following pass stores into it
        acc.fold();
    };
    auto row_of = [&](int hf) { return wg * 64 + wi * 16 + (lane >> 2) + 8 * hf; };
    auto col_of = [&](int j) { return n0 + j * 8 + 2 * (lane & 3); };

    if (!GRAD) {
        // one output parity per item, or (up-sampling layer, parity_items == 0) all four in turn
        const bool all4 = p.up && !p.parity_items;
#pragma unroll 1
        for (int q = all4 ? 0 : par; q < (all4 ? 4 : par + 1); ++q) {
            par = q, py = q >> 1, px = q & 1;
            row_classes();
            run(0);
            const float nw = (p.noise && p.noise_w) ? __ldg(p.noise_w) : 0.f;
            const bool strided = p.out_stride != 1;
            const int oh = strided ? H / 2 : Ho, ow = strided ? W / 2 : Wo;
#pragma unroll
            for (int hf = 0; hf < 2; ++hf) {
                    const int r = row_of(hf), iy = y0 + (r >> 4), ix = x0 + (r & 15);
                    if (iy >= MH || ix >= MW || (p.out_stride == 2 && ((iy | ix) & 1))) continue;
                    const int oy = iy * mul + py, ox = ix * mul + px;
                    const int cls = p.label ? region(p.label, p.ncls, ((int64_t)b * Ho + oy) * Wo + ox) : 0;
                    const float z = p.noise ? nw * __ldg(p.noise + ((int64_t)(p.noise_b == 1 ? 0 : b) * Ho + oy) * Wo + ox) : 0.f;
                    float* dst;
                    if (p.out_stride == 4)
                        dst = p.out + (((int64_t)b * oh + (iy >> 1)) * ow + (ix >> 1)) * 4 * p.nch + ((iy & 1) * 2 + (ix & 1)) * p.nch;
                    else if (strided)
                        dst = p.out + (((int64_t)b * oh + (iy >> 1)) * ow + (ix >> 1)) * p.nch;
                    else
                        dst = p.out + (((int64_t)b * Ho + oy) * Wo + ox) * p.nch;
                    if constexpr (MODE == FWD_BIAS) {
                        const float* res = p.residual ? p.residual + (dst - p.out) : nullptr;
#pragma unroll
                        for (int nf = 0; nf < NT / 8; ++nf)
                            epilogue_bias2(p, col_of(nf), acc.d[4 * nf + 2 * hf], acc.d[4 * nf + 2 * hf + 1], res, dst);
                    } else {
#pragma unroll
                        for (int nf = 0; nf < NT / 8; ++nf)
                            epilogue2<true>(p, b, cls, col_of(nf), z, acc.d[4 * nf + 2 * hf], acc.d[4 * nf + 2 * hf + 1], dst);
                    }
                }
        }
        return;
    }

    // ---- gradient: one pass per region present among the tile's source pixels (this item's share of them)
    uint32_t classes = 1u;
    if (p.label) {
        if (t == 0) s_classes = 0u;
        __syncthreads();
        uint32_t m = 0;
        const int nhalo = (TH + 2) * (TW + 2);
        for (int e = t; e < nhalo * nph_k; e += NUM_THREADS) {
            const int hp = e % nhalo, ph = ph0 + e / nhalo;
            const int sy = y0 - 1 + hp / (TW + 2), sx = x0 - 1 + hp % (TW + 2);
            if (sy >= 0 && sy < H && sx >= 0 && sx < W)
                m |= 1u << region(p.label, p.ncls, ((int64_t)b * Ho + sy * mul + (ph >> 1)) * Wo + sx * mul + (ph & 1));
        }
        m = __reduce_or_sync(0xffffffffu, m);
        if (lane == 0 && m) atomicOr(&s_classes, m);
        __syncthreads();
        classes = s_classes;
    }
#pragma unroll 1
    for (int sub = 0; sub < p.n_sub; ++sub) {           // N tiles of this work item
    n0 = it.n0 + sub * NT;
        float gxa[NR];
#pragma unroll
        for (int i = 0; i < NR; ++i) gxa[i] = 0.f;
        int k = 0;
        for (uint32_t cm = classes; cm; cm &= cm - 1, ++k) {
            if (k % p.gsplit != g) continue;
            const int c = __ffs(cm) - 1;
            run(c);
            const float* sc = p.s + ((int64_t)b * p.ncls + c) * p.nch;
#pragma unroll
            for (int nf = 0; nf < NT / 8; ++nf) {
                const int n = col_of(nf);
                const float2 s2 = __ldg(reinterpret_cast<const float2*>(sc + n));
                float gs0 = 0.f, gs1 = 0.f;
#pragma unroll
                for (int hf = 0; hf < 2; ++hf) {
                        const float u0 = acc.d[4 * nf + 2 * hf], u1 = acc.d[4 * nf + 2 * hf + 1];
                        gxa[4 * nf + 2 * hf] += s2.x * u0, gxa[4 * nf + 2 * hf + 1] += s2.y * u1;
                        if (p.gs) {
                            const int r = row_of(hf), iy = y0 + (r >> 4), ix = x0 + (r & 15);
                            if (iy < H && ix < W) {
                                const float2 xv = __ldg(reinterpret_cast<const float2*>(p.x + (((int64_t)b * H + iy) * W + ix) * p.nch + n));
                                gs0 += xv.x * u0, gs1 += xv.y * u1;
                            }
                        }
                    }
                if (p.gs) {
#pragma unroll
                    for (int o = 4; o < 32; o <<= 1) gs0 += __shfl_xor_sync(0xffffffffu, gs0, o), gs1 += __shfl_xor_sync(0xffffffffu, gs1, o);
                    if (lane < 4) {
                        float* gp = p.gs + ((int64_t)b * p.ncls + c) * p.nch + n;
                        atomicAdd(gp, gs0);
                        atomicAdd(gp + 1, gs1);
                    }
                }
            }
        }
        if (!p.out) continue;
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
                const int r = row_of(hf), iy = y0 + (r >> 4), ix = x0 + (r & 15);
                if (iy >= H || ix >= W) continue;
                float* dst = p.out + (((int64_t)b * H + iy) * W + ix) * p.nch;
#pragma unroll
                for (int nf = 0; nf < NT / 8; ++nf) {
                    const int n = col_of(nf);
                    if (p.atomic_gx) {
                        atomicAdd(dst + n, gxa[4 * nf + 2 * hf]);
                        atomicAdd(dst + n + 1, gxa[4 * nf + 2 * hf + 1]);
                    } else {
                        *reinterpret_cast<float2*>(dst + n) = make_float2(gxa[4 * nf + 2 * hf], gxa[4 * nf + 2 * hf + 1]);
                    }
                }
            }
    }
}

// ---- forward on register operands: plain layers (any mask) and (CONVT) the unmasked transposed-convolution GEMM
// The kernel above stages every operand element in shared memory as bf16 hi / lo planes and the MMAs read both operands
// from there: per K step ~112 KB cross the L1 / shared-memory data path for ~384 clocks of MMA.  Here shared memory holds
// the UNSCALED fp32 source pixels of a tile plus its 1-pixel halo (10 x 18 pixels x 32 channels, loaded once per channel
// chunk and read by all taps) and the weight tiles of every tap of the chunk, both copied by cp.async with no register
// round trip.  Each consumer thread builds its own rows of the wgmma A operand in registers: it reads the fp32 values
// at (row pixel + tap offset), multiplies them by the style of the row's own output pixel (held in registers for the
// chunk: the region does not change across taps) and splits them into bf16 hi / lo.  Only B is read from shared memory
// by the MMAs.
//
// A CTA is persistent and walks the work items blockIdx.x, + gridDim.x, ...; K runs chunk-outer, tap-inner.  A two-slot
// cp.async ring runs over the flattened (item, chunk) sequence, so the next tile's halo and weights arrive while the
// current chunk's MMAs run; one barrier per chunk.  The A fragments are double-buffered across taps: fragment set
// u = tap % 2 is rebuilt only after wgmma.wait_group has retired the MMAs of tap - 2 that read it.
// Resident weights: when the N tile's whole weight block (every chunk, every tap) fits in shared memory
// beside the two ring slots, it is copied once and stays; a slot then holds only the halo (and, at N = 32, the chunk's
// styles).  The N tile is the outermost index of an item, so a CTA reloads the block at most n_tiles - 1 times, after
// every MMA of the previous N tile has retired.  The MMAs read the same bytes in the same order either way: the results
// are bitwise identical.
// N = 128 (plain modulated layers with Cout % 128 == 0, nine taps, never resident): a chunk's weights (9 x 16 KB) do not
// fit twice.  The two slots hold only halos, and the weights stream through a ring of three slots of three taps each
// (after the halo slots, where the resident block would be) over the flattened (item, chunk, tap group) sequence: the
// next group's weights arrive while the current group's MMAs run, one barrier per group; the next chunk's halo and styles
// travel with its first group.  The slot invariant is written at the loop.  The sum order is the same as at N = 64
// (three products per K16 slice), so the results are bitwise identical to that width.
// Halo layout: pixel hp = (y + 1) * HALO_W + x + 1 at hp * 128 bytes, its 16-byte channel quad c at (c ^ (hp % 8)) * 16:
// the 8 fragment rows of a warp are 8 consecutive pixels, so the XOR spreads their reads over all 32 banks (each
// 256-byte float2 read of a warp is served in the minimal two wavefronts).
constexpr int HALO_H = TH + 2, HALO_W = TW + 2, HALO_PIX = HALO_H * HALO_W;
constexpr int HALO_BYTES = HALO_PIX * KC * 4;     // 23040

__device__ __forceinline__ void fence_frag(uint32_t (&a)[2][4]) {
#pragma unroll
    for (int i = 0; i < 8; ++i) asm volatile("" : "+r"(a[i >> 2][i & 3])::"memory");
}
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, int src_bytes) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }
// (x0, x1) -> bf16x2 hi (x0 in the low half) and the residual lo, both round-to-nearest
__device__ __forceinline__ void split2(float x0, float x1, uint32_t& hi, uint32_t& lo) {
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(hi) : "f"(x1), "f"(x0));
    const float r0 = x0 - __uint_as_float(hi << 16), r1 = x1 - __uint_as_float(hi & 0xFFFF0000u);
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(lo) : "f"(r1), "f"(r0));
}

// FWD_VOL: mosaic pixel (my, mx) of a work item in pixel-tile row ty -> its cell and the pixel (ly, lx) of the cell's
// slice; false in a gutter, off the mosaic or past the last cell (VolGrid)
__device__ __forceinline__ bool vol_cell(const Params& p, int ty, int my, int mx, int& cell, int& ly, int& lx) {
    const VolGrid& v = p.vol;
    int cy = ty * TH / p.h, cx = 0;                   // gutter 0: the tile's cell
    if (v.gutter) cy = my / (p.h + 1), cx = mx / (p.w + 1);
    ly = my - cy * (p.h + v.gutter), lx = mx - cx * (p.w + v.gutter);
    cell = cy * v.ncx + cx;
    return my >= 0 && mx >= 0 && ly >= 0 && ly < p.h && lx >= 0 && lx < p.w && cx < v.ncx && cell < v.cells;
}

// ---- transposed-convolution GEMM on register operands: all four parity classes per work item
// The unmasked layers' T' (see the up-sampling section below) is a stride-1 convolution over the 2 x 2 taps (dy, dx) in
// {0, 1}^2 with N = 4 Cout class-stacked channels, and class (a, c) uses only the taps with (dy || !a) && (dx || !c).
// A work item is 128 rows times one 32-channel slice o0 .. o0 + 31 of Cout in every class: 128 accumulator columns,
// ordered by class [(0,1), (0,0), (1,0), (1,1)].  Then every tap's classes are one contiguous column range - tap (0,0): columns 32-63, (0,1): 0-63,
// (1,0): 32-95, (1,1): 0-127 - and each tap's B tiles are one contiguous block: exactly the 9 class-tap products (ct_mma),
// no zero weights, one halo copy and four A-fragment builds per 32-channel chunk.  The accumulator starts at zero and
// every MMA accumulates, so no class needs a first-MMA flag.  Per element the sum order is chunk, tap (0,0), (0,1), (1,0),
// (1,1) (those the class uses), K16 slice, split product: that of a one-class GEMM over the class's own taps, fixed
// whatever the launch, so the output is bit reproducible.
// The B tiles of a chunk are the 32 x 32 class tiles of the w_convt_hilo planes, copied tap by tap in the column order
// ([w_hi tiles | w_lo tiles] per tap, 9 x 2 x 2 KB = 36 KB).  Resident (RES) when every chunk's 36 KB fit beside the two
// halo slots: copied once per slice (the slice is the outermost item index), else streamed with the chunk's halo.
// Rows: an 8 x 16 pixel tile of the (H + 1) x (W + 1) grid; the halo is its 9 x 17 source pixels (taps {0, 1}^2 only).
// Raw store to T' [B, H+1, W+1, 4 Cout], channel (2a + c) Cout + o.
constexpr int CT_TILE = 32 * KC * 2;                       // one 32 x 32 class tile of one bf16 plane
constexpr int CT_CHUNK = 18 * CT_TILE;                     // a chunk's 9 class tiles, both planes
constexpr int CT_HW = TW + 1, CT_HPIX = (TH + 1) * CT_HW;  // pixel-tile halo: 9 x 17
// tap k = 2 dy + dx: first column slot (of 32), slots, first tile of its weights in the chunk block
__host__ __device__ constexpr int ct_slot0(int k) { return k == 1 ? 0 : k == 3 ? 0 : 1; }
__host__ __device__ constexpr int ct_nslot(int k) { return k == 0 ? 1 : k == 3 ? 4 : 2; }
__host__ __device__ constexpr int ct_tile0(int k) { return k == 0 ? 0 : k == 1 ? 2 : k == 2 ? 6 : 10; }
__host__ __device__ constexpr int ct_class(int slot) { return slot == 0 ? 1 : slot == 1 ? 0 : slot; }

// The split products of one tap and K16 slice on its NS column slots from slot S0 (accumulator registers 16 S0 ..), B
// from bh (w_hi tiles; w_lo tiles follow): one m64n32k16 MMA per slot.  (Wider MMAs over the tap's whole column range
// would need fewer instructions, but ptxas serialises every wgmma of the kernel when register subsets of different
// widths or offsets overlap - C7511, "insufficient register resources for the wgmma pipeline"; 32-column MMAs on the four
// disjoint slots stay pipelined.)
template <int S0, int NS>
__device__ __forceinline__ void ct_mma(float (&acc)[64], const uint32_t (&hi)[4], const uint32_t (&lo)[4], uint32_t bh) {
#pragma unroll
    for (int i = 0; i < NS; ++i) {
        float (&d)[16] = *reinterpret_cast<float(*)[16]>(&acc[16 * (S0 + i)]);
        const uint32_t b = bh + i * CT_TILE;
        wgmma(d, lo, b, 1);
        wgmma(d, hi, b + NS * CT_TILE, 1);
        wgmma(d, hi, b, 1);
    }
}

template <bool RES>
__device__ __forceinline__ void convt_rs_body(const Params& p, const int items, const int stage) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~uintptr_t(127));
    const uint32_t smem_s = (uint32_t)__cvta_generic_to_shared(smem);
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5, g = lane >> 2, q = lane & 3, hc = t & 7;
    const int H = p.h, W = p.w, cout = p.nch / 4, nchunks = p.kch / KC, plane = p.nch * p.kch;
    const int halo_bytes = RES ? stage : stage - CT_CHUNK;
    const uint32_t w_s = smem_s + 2 * stage;              // resident weight block: chunk kc at w_s + kc * CT_CHUNK

    // work item: pixel tile (tx, ty), sample b, slice n0 .. n0 + 31 of Cout (the outermost index)
    auto decode = [&](int idx) { return decode_item<false>(p, idx, 32); };
    // this thread's fragment rows g, g + 8 of tile row `warp`: halo offsets of their tap (0,0) source pixels
    const int hb[2] = {warp * CT_HW + g, warp * CT_HW + g + 8};
    // this thread's styles of chunk kc: its fragment channels (one style per sample)
    auto load_styles = [&](const Item& it, int kc, float2 (&sv)[4]) {
#pragma unroll
        for (int j = 0; j < 4; ++j) sv[j] = __ldg(reinterpret_cast<const float2*>(p.s + it.b * p.kch + kc * KC + 8 * j + 2 * q));
    };
    // the 18 (class tile, plane) pairs of chunk kc of slice o0 at dst: copy e of the chunk is pair e / 128, row
    // 8 (c / 32) + c % 8 and channel quad (c / 8) % 4 of the tile (c = e % 128), byte 16 c of the tile
    auto copy_weights = [&](int o0, int kc, uint32_t dst) {
#pragma unroll
        for (int i = 0; i < 18 * 128 / NUM_THREADS; ++i) {
            const int e = t + NUM_THREADS * i, u = e >> 7, c = e & 127;
            const int k = u < 2 ? 0 : u < 6 ? 1 : u < 10 ? 2 : 3, ns = ct_nslot(k), w = u - ct_tile0(k);
            const int hl = w >= ns, cls = ct_class(ct_slot0(k) + w - hl * ns);
            const int n = cls * cout + o0 + (c >> 5) * 8 + (c & 7);
            cp_async16(dst + e * 16, p.wt + (hl * 9 + (k >> 1) * 3 + (k & 1)) * plane + n * p.kch + kc * KC + ((c >> 3) & 3) * 8, 16);
        }
    };
    auto copy_block = [&](int o0) {
#pragma unroll 1
        for (int kc = 0; kc < nchunks; ++kc) copy_weights(o0, kc, w_s + kc * CT_CHUNK);
    };
    // ring slot buf <- chunk kc of the item's halo (zero outside the image) and, streaming, its weights
    auto prefetch = [&](const Item& it, int kc, int buf) {
        const uint32_t st = smem_s + buf * stage;
        const float* xb = p.a + (int64_t)it.b * H * W * p.kch + kc * KC + hc * 4;
        const int sy0 = it.ty * TH - 1, sx0 = it.tx * TW - 1;
#pragma unroll
        for (int i = 0; i < (CT_HPIX * 8 + NUM_THREADS - 1) / NUM_THREADS; ++i) {
            const int hp = (t >> 3) + 32 * i;
            if (hp < CT_HPIX) {
                const int hy = hp / CT_HW, sy = sy0 + hy, sx = sx0 + hp - hy * CT_HW;
                const bool ok = sy >= 0 && sy < H && sx >= 0 && sx < W;
                cp_async16(st + hp * 128 + ((hc ^ (hp & 7)) << 4), ok ? xb + (sy * W + sx) * p.kch : p.a, ok ? 16 : 0);
            }
        }
        if (!RES) copy_weights(it.n0, kc, st + halo_bytes);
        cp_async_commit();
    };

    float acc[64];
    uint32_t fh[2][2][4], fl[2][2][4];                    // [tap % 2][K16 slice][register]: x_hi, x_lo fragments
    // fragment register r of slice ks: row g + 8 (r & 1) of the thread's rows, channels 16 ks + 8 (r >> 1) + 2 q, + 1
    auto build = [&](const uint8_t* halo, int toff, const float2 (&sv)[4], uint32_t (&hi)[2][4], uint32_t (&lo)[2][4]) {
#pragma unroll
        for (int ks = 0; ks < 2; ++ks)
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                const int j = 2 * ks + (r >> 1), hp = hb[r & 1] + toff;
                const float2 v = *reinterpret_cast<const float2*>(halo + hp * 128 + (((2 * j + (q >> 1)) ^ (hp & 7)) << 4) + (q & 1) * 8);
                split2(v.x * sv[j].x, v.y * sv[j].y, hi[ks][r], lo[ks][r]);
            }
    };
    // tap K's MMAs, both K16 slices, B from bt (its tiles in the chunk block)
    auto issue = [&](auto kk, uint32_t bt, uint32_t (&hi)[2][4], uint32_t (&lo)[2][4]) {
        constexpr int K = decltype(kk)::value;
        fence_regs(acc);
        fence_frag(hi);
        fence_frag(lo);
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < 2; ++ks) ct_mma<ct_slot0(K), ct_nslot(K)>(acc, hi[ks], lo[ks], bt + ct_tile0(K) * CT_TILE + ks * 2 * LBO);
        wgmma_commit();
        fence_regs(acc);
        fence_frag(hi);
        fence_frag(lo);
    };
    auto store_item = [&](const Item& it) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int iy = it.ty * TH + warp, ix = it.tx * TW + g + 8 * h;
            if (iy > H || ix > W) continue;
            float* dst = p.out + (((int64_t)it.b * (H + 1) + iy) * (W + 1) + ix) * p.nch;
#pragma unroll
            for (int nf = 0; nf < 16; ++nf)
                *reinterpret_cast<float2*>(dst + ct_class(nf >> 2) * cout + it.n0 + (nf & 3) * 8 + 2 * q) =
                    make_float2(acc[4 * nf + 2 * h], acc[4 * nf + 2 * h + 1]);
        }
    };

    int item = blockIdx.x;
    if (item >= items) return;
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    Item cur = decode(item), nxt;
    float2 sty[4], sty_n[4];
    load_styles(cur, 0, sty);
    int kc = 0, buf = 0;
    if (RES) copy_block(cur.n0);                          // committed with the first halo
    prefetch(cur, 0, 0);
#pragma unroll 1
    while (true) {
        const bool last_chunk = kc == nchunks - 1;
        const int item_n = last_chunk ? item + (int)gridDim.x : item, kc_n = last_chunk ? 0 : kc + 1;
        const bool more = item_n < items;
        // slot buf complete and visible to the async proxy; every MMA of the previous chunk retired (wait_group 0 below),
        // so the other slot may be refilled once this chunk's first MMAs are issued.  Fragment set k % 2 is rebuilt
        // after wait_group 1 has retired tap k - 2, its last reader.
        cp_async_wait_all();
        fence_proxy_async();
        __syncthreads();
        const uint8_t* halo = smem + buf * stage;
        const uint32_t bt = RES ? w_s + kc * CT_CHUNK : smem_s + buf * stage + halo_bytes;
        build(halo, 0, sty, fh[0], fl[0]);
        issue(std::integral_constant<int, 0>{}, bt, fh[0], fl[0]);
        if (more) {                                       // while tap (0,0)'s MMAs run
            nxt = last_chunk ? decode(item_n) : cur;
            prefetch(nxt, kc_n, buf ^ 1);
            load_styles(nxt, kc_n, sty_n);
        }
        build(halo, 1, sty, fh[1], fl[1]);
        issue(std::integral_constant<int, 1>{}, bt, fh[1], fl[1]);
        wgmma_wait<1>();
        build(halo, CT_HW, sty, fh[0], fl[0]);
        issue(std::integral_constant<int, 2>{}, bt, fh[0], fl[0]);
        wgmma_wait<1>();
        build(halo, CT_HW + 1, sty, fh[1], fl[1]);
        issue(std::integral_constant<int, 3>{}, bt, fh[1], fl[1]);
        wgmma_wait<0>();
        fence_regs(acc);
        if (RES && more && nxt.n0 != cur.n0) {            // next slice: its block, once both warpgroups' MMAs retired;
            __syncthreads();                              // the barrier at the top of the loop waits for the copies
            copy_block(nxt.n0);
            cp_async_commit();
        }
        if (last_chunk) {
            store_item(cur);
#pragma unroll
            for (int i = 0; i < 64; ++i) acc[i] = 0.f;
        }
        if (!more) break;
        cur = nxt, item = item_n, kc = kc_n, buf ^= 1;
#pragma unroll
        for (int j = 0; j < 4; ++j) sty[j] = sty_n[j];
    }
}

// ---- masked transposed-convolution GEMM on register operands (ROWS): gathered rows, one parity class per work item
// The masked layers' T' rows are (T' pixel, region) pairs from a row list (p.rows, see the masked up-sampling section
// below), so there is no pixel tile to share a halo.  A work item is one 128-row block rb of sample b's list times NT
// channels n0 .. of ONE class cls (columns cls Cout + ..): K runs over the class's taps in the order {0, 1, 3, 4} (those
// it uses: 4 >> popcount(cls) of them) and, inside each tap, the 32-channel chunks - tap-outer, chunk-inner.  A K step
// (tap, chunk) stages the 128 rows' source pixels at the tap's offset (16-byte cp.async copies, zero off the grid and past
// the list's end; the quads swizzled as in the halo) and the step's NT x 32 weight tiles; each consumer thread builds its
// fragment rows from them scaled by the style of the row's own region (read per step from the style table), splits them
// (split2) and issues split_mma.  Per element the sum order is tap, chunk, K16 slice, split product - whatever NT is
// (64 and 128 give the same bits), so a face's output does not depend on the batch it is in.
// A slot of the two-slot cp.async ring holds p.ntaps consecutive K steps ([A tiles | B tiles]); the ring runs over the
// flattened (item, step group) sequence, one barrier per group, and the fragments are double-buffered across steps as in
// the plain mode.
// Schedule: the items of the launch are those of the row blocks holding rows (blocks past a sample's row count, and every
// block of a sample whose list overflowed, row_count > cap, have none), in the order sample, row block, class, slice.
// Every row block carries the same 9 nchunks Cout / NT K steps, so each CTA computes from the row counts where its equal
// share of the launch's steps begins and ends and takes the items that start inside it: the chains of 4, 2, 2 and 1 taps
// balance over the CTAs, and a CTA runs all classes of a row block back to back, sharing its gathered rows in L2.  Raw
// store to T'c [B, cap, 4 Cout] (rows below the count).
struct RowItem {
    int b, rb, cls, n0, cnt, nsteps;
};
// item k (class k / slices, slice k % slices) of row block rb of sample b, starting at step s of the launch
struct RowPos {
    int b, rb, k;
    int64_t s;
};
template <int NT>
__device__ __forceinline__ void rows_rs_body(const Params& p, const int stage) {
    constexpr int A_TILE = M * KC * 4, B_PLANE = NT * KC * 2, B_CP = B_PLANE / 16;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~uintptr_t(127));
    const uint32_t smem_s = (uint32_t)__cvta_generic_to_shared(smem);
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5, g = lane >> 2, q = lane & 3, hc = t & 7;
    const int H = p.h, W = p.w, cout = p.nch / 4, nchunks = p.kch / KC, plane = p.nch * p.kch, spg = p.ntaps;
    const int w_ofs = spg * A_TILE;                       // B tiles of a slot: step k at w_ofs + 2 k B_PLANE

    const int nsl = p.n_tiles;
    // row blocks of sample b holding rows
    auto blocks_of = [&](int b) {
        const int c = __ldg(p.row_count + b);
        return c <= p.cap ? (c + M - 1) / M : 0;
    };
    // this CTA's share [lo, hi) of the launch's K steps
    int64_t nblk = 0;
    for (int b = 0; b < p.batch; ++b) nblk += blocks_of(b);
    const int64_t per_block = 9ll * nchunks * nsl, total = nblk * per_block;
    const int64_t lo = total * blockIdx.x / gridDim.x, hi = total * (blockIdx.x + 1) / gridDim.x;
    auto decode = [&](const RowPos& q) {
        RowItem it;
        it.b = q.b, it.rb = q.rb, it.cls = q.k / nsl;
        it.n0 = it.cls * cout + (q.k - it.cls * nsl) * NT;
        it.cnt = __ldg(p.row_count + q.b);
        it.nsteps = (4 >> __popc(it.cls)) * nchunks;
        return it;
    };
    // the item after q: next slice, class, row block holding rows, sample
    auto advance = [&](RowPos q) {
        q.s += (4 >> __popc(q.k / nsl)) * nchunks;
        if (++q.k == 4 * nsl) {
            q.k = 0;
            if (++q.rb == blocks_of(q.b)) {
                q.rb = 0;
                do ++q.b;
                while (q.b < p.batch && blocks_of(q.b) == 0);
            }
        }
        return q;
    };
    auto mine = [&](const RowPos& q) { return q.b < p.batch && q.s < hi; };
    // K step s of the item: tap ti = s / nchunks of its class (offset (dy, dx)), chunk s % nchunks
    auto step_tap = [&](const RowItem& it, int s, int& dy, int& dx) {
        const int ti = s / nchunks;
        if (it.cls & 2) dy = 1, dx = (it.cls & 1) ? 1 : ti;
        else if (it.cls & 1) dy = ti, dx = 1;
        else dy = ti >> 1, dx = ti & 1;
    };
    // the item's rows this thread gathers, (t >> 3) + 32 i: packed positions, valid where i < vcnt (loaded once per item,
    // before its first copies)
    uint32_t rv[4];
    int vcnt = 0;
    // ring slot buf <- step group gi of the item: per step the gathered rows (row r at r * 128 bytes) and both weight planes
    auto prefetch = [&](const RowItem& it, int gi, int buf) {
        if (gi == 0) {
            vcnt = 0;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int r = it.rb * M + (t >> 3) + 32 * i;
                rv[i] = r < it.cnt ? __ldg(p.rows + (int64_t)it.b * p.cap + r) : 0u;
                vcnt += r < it.cnt;
            }
        }
        const uint32_t st = smem_s + buf * stage;
        const int s0 = gi * spg, ns = min(spg, it.nsteps - s0);
        for (int k = 0; k < ns; ++k) {
            const int s = s0 + k, kc = s % nchunks;
            int dy, dx;
            step_tap(it, s, dy, dx);
            const float* xb = p.a + (int64_t)it.b * H * W * p.kch + kc * KC + hc * 4;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int r = (t >> 3) + 32 * i;
                const int sy = (int)(rv[i] >> (ROW_NBITS + 5)) + dy - 1, sx = (int)((rv[i] >> 5) & ((1u << ROW_NBITS) - 1)) + dx - 1;
                const bool ok = i < vcnt && sy >= 0 && sy < H && sx >= 0 && sx < W;
                cp_async16(st + k * A_TILE + r * 128 + ((hc ^ (r & 7)) << 4), ok ? xb + (sy * W + sx) * p.kch : p.a, ok ? 16 : 0);
            }
            // copy c of a plane: row 8 (c / 32) + c % 8, channel quad (c / 8) % 4 of the tile, byte 16 c
            const int tap = dy * 3 + dx;
            const uint32_t bd = st + w_ofs + k * 2 * B_PLANE;
#pragma unroll
            for (int c = t; c < B_CP; c += NUM_THREADS) {
                const __nv_bfloat16* wb = p.wt + (it.n0 + (c >> 5) * 8 + (c & 7)) * p.kch + kc * KC + ((c >> 3) & 3) * 8;
                cp_async16(bd + c * 16, wb + tap * plane, 16);
                cp_async16(bd + B_PLANE + c * 16, wb + (9 + tap) * plane, 16);
            }
        }
        cp_async_commit();
    };
    // regions of this thread's fragment rows 16 warp + g, + 8
    auto row_regions = [&](const RowItem& it, int (&c)[2]) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int i = it.rb * M + warp * 16 + g + 8 * h;
            c[h] = i < it.cnt ? min((int)(__ldg(p.rows + (int64_t)it.b * p.cap + i) & 31u), p.ncls - 1) : 0;
        }
    };
    // styles of step s's chunk at this thread's fragment channels, per fragment row's region
    auto load_styles = [&](const RowItem& it, const int (&c)[2], int s, float2 (&sv)[2][4]) {
        const int kc = s % nchunks;
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int j = 0; j < 4; ++j)
                sv[h][j] = __ldg(reinterpret_cast<const float2*>(p.s + (it.b * p.ncls + c[h]) * p.kch + kc * KC + 8 * j + 2 * q));
    };

    SplitAcc<NT> acc{};                                   // zero: the fences read every register
    uint32_t fh[2][2][4], fl[2][2][4];                    // [step % 2][K16 slice][register]: x_hi, x_lo fragments
    // fragments of a step from its A tile and styles: register r of slice ks is row g + 8 (r & 1), channels
    // 16 ks + 8 (r >> 1) + 2 q, + 1
    auto build = [&](const uint8_t* a, const float2 (&sv)[2][4], uint32_t (&hi)[2][4], uint32_t (&lo)[2][4]) {
#pragma unroll
        for (int ks = 0; ks < 2; ++ks)
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                const int h = r & 1, j = 2 * ks + (r >> 1), hp = warp * 16 + g + 8 * h;
                const float2 v = *reinterpret_cast<const float2*>(a + hp * 128 + (((2 * j + (q >> 1)) ^ (hp & 7)) << 4) + (q & 1) * 8);
                split2(v.x * sv[h][j].x, v.y * sv[h][j].y, hi[ks][r], lo[ks][r]);
            }
    };
    auto issue = [&](uint32_t bt, uint32_t (&hi)[2][4], uint32_t (&lo)[2][4], bool first_mma) {
        acc.fence();
        fence_frag(hi);
        fence_frag(lo);
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < 2; ++ks) {
            const uint32_t bh = bt + ks * 2 * LBO;
            split_mma(acc, hi[ks], lo[ks], bh, bh + B_PLANE, (first_mma && ks == 0) ? 0 : 1);
        }
        wgmma_commit();
        acc.fence();
        fence_frag(hi);
        fence_frag(lo);
    };
    auto store_item = [&](const RowItem& it) {
        acc.fold();
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int i = it.rb * M + warp * 16 + g + 8 * h;
            if (i >= it.cnt) continue;
            float* dst = p.out + ((int64_t)it.b * p.cap + i) * p.nch + it.n0 + 2 * q;
#pragma unroll
            for (int nf = 0; nf < NT / 8; ++nf)
                *reinterpret_cast<float2*>(dst + nf * 8) = make_float2(acc.d[4 * nf + 2 * h], acc.d[4 * nf + 2 * h + 1]);
        }
    };

    // the first item starting at or after lo: in row block lo / per_block (the n-th holding rows), else the next one
    RowPos pos{0, 0, 0, lo - lo % per_block};
    for (int64_t n = lo / per_block; pos.b < p.batch; ++pos.b) {
        const int nb = blocks_of(pos.b);
        if (n < nb) {
            pos.rb = (int)n;
            break;
        }
        n -= nb;
    }
    while (pos.s < lo) pos = advance(pos);
    if (!mine(pos)) return;
    RowPos pos_n = advance(pos);
    RowItem cur = decode(pos), nxt;
    int cls[2], cls_n[2];
    row_regions(cur, cls);
    float2 sty[2][4];                                     // styles of the next step to build
    load_styles(cur, cls, 0, sty);
    int gi = 0, buf = 0;
    prefetch(cur, 0, 0);
#pragma unroll 1
    while (true) {
        const bool last_group = (gi + 1) * spg >= cur.nsteps;
        const int gi_n = last_group ? 0 : gi + 1;
        const bool more = !last_group || mine(pos_n);
        // slot buf complete and visible to the async proxy; every MMA of the previous group retired (wait_group 0 below),
        // so the other slot may be refilled once this group's first MMAs are issued.  Fragment set k % 2 is rebuilt
        // after wait_group 1 has retired step k - 2, its last reader.
        cp_async_wait_all();
        fence_proxy_async();
        __syncthreads();
        const uint8_t* a_slot = smem + buf * stage;
        const uint32_t b_slot = smem_s + buf * stage + w_ofs;
        const int s0 = gi * spg, ns = min(spg, cur.nsteps - s0);
#pragma unroll 1
        for (int k = 0; k < ns; k += 2) {
            if (k >= 2) wgmma_wait<1>();
            build(a_slot + k * A_TILE, sty, fh[0], fl[0]);
            if (s0 + k + 1 < cur.nsteps) load_styles(cur, cls, s0 + k + 1, sty);
            issue(b_slot + k * 2 * B_PLANE, fh[0], fl[0], s0 + k == 0);
            if (k + 1 < ns) {
                wgmma_wait<1>();
                build(a_slot + (k + 1) * A_TILE, sty, fh[1], fl[1]);
                if (s0 + k + 2 < cur.nsteps) load_styles(cur, cls, s0 + k + 2, sty);
                issue(b_slot + (k + 1) * 2 * B_PLANE, fh[1], fl[1], false);
            }
            if (k == 0 && more) {                         // once the group's first two steps are queued
                if (last_group) {
                    nxt = decode(pos_n);
                    row_regions(nxt, cls_n);
                } else {
                    nxt = cur, cls_n[0] = cls[0], cls_n[1] = cls[1];
                }
                prefetch(nxt, gi_n, buf ^ 1);
            }
        }
        wgmma_wait<0>();
        acc.fence();
        if (last_group) store_item(cur);
        if (!more) break;
        if (last_group) {
            cur = nxt, cls[0] = cls_n[0], cls[1] = cls_n[1];
            pos_n = advance(pos_n);
            load_styles(cur, cls, 0, sty);
        }
        gi = gi_n, buf ^= 1;
    }
}

// Work items: (pixel tile, sample, N tile) (decode_item).  p.out_stride == 1, no up-sampling, no shift: the plain
// modulated convolution (epilogue: per-region demodulation, noise, bias, activation).  RES: resident weights - a
// compile-time choice, so that the streaming instantiation carries none of the resident mode's code.  stage: bytes of one ring slot, [halo | tap 0 w_hi | w_lo |
// tap 1 ...] when the weights stream, [halo] when resident or at N = 128 (the weight block follows the two slots: (chunk kc, tap ti)
// at (kc * ntaps + ti) * B_TAP).  Resident at N = 32 the kernel is compiled for two CTAs per SM (<= 128 registers): the
// next chunk's styles (its 32 channels of every region of the item's sample) wait in the slot after the halo instead of
// in registers.  Index arithmetic is 32-bit (the host checks the item count; a sample's activations and the weight
// planes stay below 2^31 elements), and the next (item, chunk) is decoded once, when its copies are issued.
// DENSE (compile time, like RES): the plain convolution of ESRGAN's networks - no styles, labels or regions (the A
// fragments are the unscaled source values), the input read and the output written with pixel pitches p.a_ld / p.out_ld
// (channel slices of wider buffers: a residual dense block keeps x, x1 .. x4 in one [B, H, W, 160] buffer and its convs
// read and write disjoint channel ranges of it), optionally nearest 2x up-sampling in the halo copy, and epilogue_dense2.
// REFL (DENSE only, compile time): the halo outside the grid is the reflection padding of p.reflect instead of zero - GPEN's
// ParseNet; the zero-fill instantiations carry none of its code.
// PW (DENSE only, compile time): the 1x1 convolution.  There is no halo: the 128 rows of an item are its 128 output pixels,
// read at (in_stride y, in_stride x) of the input, so a stride-2 shortcut needs no space-to-depth pass.  The tap loop runs
// over the p.ntaps 32-channel K chunks of a ring slot instead (slot: ntaps tiles of 128 pixels x 32 channels, then their
// ntaps weight tiles; K chunk c of the layer is tile c % ntaps of step c / ntaps), so one copy and one barrier cover
// 2 ntaps K16 slices.  Weights [2][Cout][Cin]; epilogue_pw2.
// VOL (DENSE only, compile time): the 3x3x3 convolution of face-vid2vid's 3D blocks over [B, H, W, D, Cin] -> [B, H, W, D,
// Cout] (pixel pitches p.a_ld = D Cin, p.out_ld = D Cout; H, W = p.h, p.w, the output grid).  The pixel tiles cover the
// mosaic p.vol (VolGrid, p.mh x p.mw, p.batch = 1): the halo copy maps each mosaic pixel to (cell, y, x), the cell to
// (b, z), and reads K chunk kc at depth z + kc / (Cin / 32) - 1, zero in gutters, past the last cell and outside the
// depth range; the store skips gutters.  Weights [2][9][Cout][3 Cin] (kz-major K); p.up is the (1, 2, 2) nearest
// up-sampling.  The zero-fill 2D instantiations carry none of its code.
template <int NT, bool RES, bool DENSE = false, bool REFL = false, bool PW = false, bool VOL = false, bool CONVT = false,
          int EPI = EPI_PLAIN, bool ROWS = false>
__global__ void __launch_bounds__(NUM_THREADS, (NT == 32 && RES) ? 2 : 1)
    conv3x3_rs_kernel(const __grid_constant__ Params p, const int items, const int stage) {
    static_assert(NT == 32 || NT == 64 || (NT == 128 && (CONVT || (!RES && !DENSE))), "register-operand forward: N tiles of 32, 64 or 128");
    static_assert(!CONVT || (NT == 128 && !DENSE), "transposed-convolution form: 128 accumulator columns, modulated");
    static_assert(!ROWS || (!RES && !DENSE && !CONVT), "gathered rows: modulated, streamed weights");
    if constexpr (CONVT) {
        convt_rs_body<RES>(p, items, stage);
        return;
    }
    if constexpr (ROWS) {
        rows_rs_body<NT>(p, stage);
        return;
    }
    static_assert(!REFL || DENSE, "reflection padding: plain mode only");
    static_assert(!PW || (DENSE && !REFL), "pointwise: plain mode, zero padding");
    static_assert(!VOL || (DENSE && !REFL && !PW), "volumetric: plain mode, zero padding");
    static_assert(EPI != EPI_SPADE || (DENSE && !REFL && !PW && !VOL), "SPADE epilogue: plain mode, zero padding");
    static_assert(EPI != EPI_FACTOR || PW, "per-pixel factor: pointwise mode");
    constexpr int PW_TILE = M * KC * 4;                   // PW: one K chunk of the item's 128 pixels
    constexpr int B_PLANE = NT * KC * 2, B_TAP = 2 * B_PLANE;
    constexpr int B_CP = B_PLANE / 16;                    // 16-byte copies per (tap, plane)
    constexpr int B_PPI = B_CP < NUM_THREADS ? NUM_THREADS / B_CP : 1;    // (tap, plane) pairs per pass of the threads
    constexpr int TG = 3, W_SLOT = TG * B_TAP;            // N = 128: taps per weight-ring slot
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~uintptr_t(127));
    const uint32_t smem_s = (uint32_t)__cvta_generic_to_shared(smem);
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    // this thread's fragment rows: tile row `warp`, columns g and g + 8; fragment channels 8 j + 2 q, + 1 (j = 2 ks + half)
    const int g = lane >> 2, q = lane & 3;
    const int nchunks = p.kch / (PW ? KC * p.ntaps : KC), plane = p.nch * p.kch;
    const int H = p.h, W = p.w, MH = p.mh, MW = p.mw;
    // this thread's copies: channel quad t % 8 of halo pixels t / 8 + 32 i; weight row bn, quad bkq of the (tap, plane)
    // pairs bpl + B_PPI k
    const int hc = t & 7, bc = t % B_CP, bpl = t / B_CP;
    const int bn = (bc >> 5) * 8 + (bc & 7), bkq = (bc >> 3) & 3;
    const uint32_t b_dst = (bn >> 3) * SBO + bkq * LBO + (bn & 7) * 16;
    // where the next chunk's styles wait: in the ring slot (resident at N = 32) or in registers, loaded while the current
    // chunk's MMAs run
    constexpr bool STY_SMEM = NT == 32 && RES && !DENSE, STY_REG = !STY_SMEM && !DENSE;
    const int sty_ofs = PW ? p.ntaps * PW_TILE : HALO_BYTES, w_ofs = sty_ofs + (STY_SMEM ? p.ncls * KC * 4 : 0);    // in a ring slot
    const uint32_t w_s = smem_s + 2 * stage;              // resident weight block

    // region of each fragment row's own output pixel
    auto row_classes = [&](const Item& it, int (&c)[2]) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int iy = it.ty * TH + warp, ix = it.tx * TW + g + 8 * h;
            c[h] = (p.label && iy < MH && ix < MW) ? region(p.label, p.ncls, ((int64_t)it.b * MH + iy) * MW + ix) : 0;
        }
    };
    // this thread's styles of chunk kc (from ring slot `buf` when STY_SMEM): the fragment channels of each row's region
    auto load_styles = [&](const Item& it, int kc, int buf, const int (&c)[2], float2 (&sv)[2][4]) {
        const float* tab = STY_SMEM ? reinterpret_cast<const float*>(smem + buf * stage + sty_ofs)
                                    : p.s + (it.b * p.ncls) * p.kch + kc * KC;
        const int ld = STY_SMEM ? KC : p.kch;
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float2* v = reinterpret_cast<const float2*>(tab + c[h] * ld + 8 * j + 2 * q);
                sv[h][j] = STY_SMEM ? *v : __ldg(v);
            }
    };
    // weight tiles of chunk kc of the item's taps in the no-swizzle K-major core-matrix layout, tap ti at dst + ti * B_TAP
    auto copy_weights = [&](const Item& it, int kc, uint32_t dst) {
        const __nv_bfloat16* wb = p.wt + (it.n0 + bn) * p.kch + kc * KC + bkq * 8;
        for (int pl = bpl; pl < 2 * p.ntaps; pl += B_PPI) {
            const int ti = pl >> 1, hl = pl & 1;
            if constexpr (PW)
                cp_async16(dst + b_dst + ti * B_TAP + hl * B_PLANE, wb + hl * plane + (kc * (p.ntaps - 1) + ti) * KC, 16);
            else
                cp_async16(dst + b_dst + ti * B_TAP + hl * B_PLANE, wb + (hl * 9 + p.taps[ti]) * plane, 16);
        }
    };
    // the N tile's resident block: chunk kc's taps at w_s + kc * ntaps * B_TAP
    auto copy_block = [&](const Item& it) {
#pragma unroll 1
        for (int kc = 0; kc < nchunks; ++kc) copy_weights(it, kc, w_s + kc * p.ntaps * B_TAP);
    };
    // N = 128: weight-ring slot ws <- taps TG tg .. of chunk kc.  Copy c of a (tap, plane) is row 8 (c / 32) + c % 8,
    // channel quad (c / 8) % 4 of the tile: byte 16 c of the plane in the core-matrix layout
    auto copy_group = [&](const Item& it, int kc, int tg, int ws) {
        if constexpr (NT == 128) {
#pragma unroll
            for (int c = t; c < B_CP; c += NUM_THREADS) {
                const __nv_bfloat16* wb = p.wt + (it.n0 + (c >> 5) * 8 + (c & 7)) * p.kch + kc * KC + ((c >> 3) & 3) * 8;
#pragma unroll
                for (int pl = 0; pl < 2 * TG; ++pl)
                    cp_async16(w_s + ws * W_SLOT + pl * B_PLANE + c * 16, wb + ((pl & 1) * 9 + p.taps[TG * tg + (pl >> 1)]) * plane, 16);
            }
        }
    };
    // ring slot `buf` <- (item, chunk): the halo with zero fill outside the image (the convolution's padding) and the styles
    auto copy_halo = [&](const Item& it, int kc, int buf) {
        const uint32_t st = smem_s + buf * stage;
        if constexpr (PW) {
            // tile ti of the slot: K chunk kc * ntaps + ti of the item's pixels (pixel e = 16 row + column at e * 128 bytes,
            // the quads swizzled as in the halo); pixels off the output grid are zero-filled
            const float* xb = p.a + (int64_t)it.b * H * W * p.a_ld + kc * p.ntaps * KC + hc * 4;
            for (int e = t >> 3; e < p.ntaps * M; e += NUM_THREADS / 8) {
                const int ti = e / M, r = e % M, iy = it.ty * TH + (r >> 4), ix = it.tx * TW + (r & 15);
                const bool ok = iy < MH && ix < MW;
                const float* src = xb + (iy * p.in_stride * W + ix * p.in_stride) * p.a_ld + ti * KC;
                cp_async16(st + e * 128 + ((hc ^ (e & 7)) << 4), ok ? src : p.a, ok ? 16 : 0);
            }
            return;
        }
        const int sy0 = it.ty * TH - 1, sx0 = it.tx * TW - 1;
        if constexpr (VOL) {
            const int cin = p.kch / 3, nc = cin / KC, dz = kc / nc - 1, us = p.up, SH = H >> us, SW = W >> us;
            const float* xc = p.a + (kc - (dz + 1) * nc) * KC + hc * 4;
#pragma unroll
            for (int i = 0; i < (HALO_PIX * 8 + NUM_THREADS - 1) / NUM_THREADS; ++i) {
                const int hp = (t >> 3) + 32 * i;
                if (hp < HALO_PIX) {
                    const int hy = hp / HALO_W;
                    int cell, ly, lx;
                    bool ok = vol_cell(p, it.ty, sy0 + hy, sx0 + hp - hy * HALO_W, cell, ly, lx);
                    const int b = cell / p.vol.depth, z = cell - b * p.vol.depth + dz;
                    ok = ok && z >= 0 && z < p.vol.depth;
                    const float* src = xc + ((int64_t)(b * SH + (ly >> us)) * SW + (lx >> us)) * p.a_ld + z * p.vox_in;
                    cp_async16(st + hp * 128 + ((hc ^ (hp & 7)) << 4), ok ? src : p.a, ok ? 16 : 0);
                }
            }
            return;
        }
        // DENSE with up-sampling: the source image is (H / 2) x (W / 2), pixel (sy, sx) of the grid reads (sy >> 1, sx >> 1)
        const int ld = DENSE ? p.a_ld : p.kch, us = DENSE ? p.up : 0, SW = W >> us;
        const float* xb = p.a + (int64_t)it.b * (H >> us) * SW * ld + kc * KC + hc * 4;
#pragma unroll
        for (int i = 0; i < (HALO_PIX * 8 + NUM_THREADS - 1) / NUM_THREADS; ++i) {
            const int hp = (t >> 3) + 32 * i;
            if (hp < HALO_PIX) {
                const int hy = hp / HALO_W, sy = sy0 + hy, sx = sx0 + hp - hy * HALO_W;
                if constexpr (REFL) {
                    // mirror (p.reflect == 1) or replicate, then clamp: pixels past a partial tile's edge stay in the
                    // image (they feed only outputs that are not stored)
                    int ry = sy, rx = sx;
                    if (p.reflect == 1) {
                        ry = sy < 0 ? -sy : (sy >= H ? 2 * H - 2 - sy : sy);
                        rx = sx < 0 ? -sx : (sx >= W ? 2 * W - 2 - sx : sx);
                    }
                    ry = min(max(ry, 0), H - 1), rx = min(max(rx, 0), W - 1);
                    cp_async16(st + hp * 128 + ((hc ^ (hp & 7)) << 4), xb + ((ry >> us) * SW + (rx >> us)) * ld, 16);
                } else {
                    const bool ok = sy >= 0 && sy < H && sx >= 0 && sx < W;
                    cp_async16(st + hp * 128 + ((hc ^ (hp & 7)) << 4), ok ? xb + ((sy >> us) * SW + (sx >> us)) * ld : p.a, ok ? 16 : 0);
                }
            }
        }
        if (STY_SMEM && t < p.ncls * (KC / 4))                        // ncls <= 32: one 16-byte copy per thread at most
            cp_async16(st + sty_ofs + t * 16, p.s + (it.b * p.ncls + (t >> 3)) * p.kch + kc * KC + (t & 7) * 4, 16);
    };
    // ... then, unless the weights are resident, the weight tiles of the item's taps (N = 128: of its first tap group,
    // into weight-ring slot ws)
    int ws = 0;
    auto prefetch = [&](const Item& it, int kc, int buf) {
        copy_halo(it, kc, buf);
        if constexpr (NT == 128)
            copy_group(it, kc, 0, ws);
        else if (!RES)
            copy_weights(it, kc, smem_s + buf * stage + w_ofs);
        cp_async_commit();
    };

    SplitAcc<NT> acc{};                               // zero: the fences read every register
    uint32_t fh[2][2][4], fl[2][2][4];                    // [tap % 2][K16 slice][register]: x_hi, x_lo fragments

    // fragment register r of slice ks: row g + 8 (r & 1), channels 16 ks + 8 (r >> 1) + 2 q, + 1
    auto build = [&](const uint8_t* halo, int tap, const float2 (&sv)[2][4], uint32_t (&hi)[2][4], uint32_t (&lo)[2][4]) {
        const int dy = tap / 3, dx = tap % 3;
#pragma unroll
        for (int ks = 0; ks < 2; ++ks)
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                const int h = r & 1, j = 2 * ks + (r >> 1);
                const int hp = PW ? tap * M + warp * TW + g + 8 * h : (warp + dy) * HALO_W + g + 8 * h + dx;
                const float2 v = *reinterpret_cast<const float2*>(halo + hp * 128 + (((2 * j + (q >> 1)) ^ (hp & 7)) << 4) + (q & 1) * 8);
                if constexpr (DENSE)
                    split2(v.x, v.y, hi[ks][r], lo[ks][r]);
                else
                    split2(v.x * sv[h][j].x, v.y * sv[h][j].y, hi[ks][r], lo[ks][r]);
            }
    };
    auto issue = [&](uint32_t bt, uint32_t (&hi)[2][4], uint32_t (&lo)[2][4], bool first_mma) {
        acc.fence();
        fence_frag(hi);
        fence_frag(lo);
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < 2; ++ks) {
            const uint32_t bh = bt + ks * 2 * LBO, bl = bh + B_PLANE;
            const int accumulate = (first_mma && ks == 0) ? 0 : 1;
            split_mma(acc, hi[ks], lo[ks], bh, bl, accumulate);
        }
        wgmma_commit();
        acc.fence();
        fence_frag(hi);
        fence_frag(lo);
    };

    // epilogue of an item: this thread's two rows of the tile, NT / 8 channel pairs each
    auto store_item = [&](const Item& it, const int (&c)[2]) {
        acc.fold();
        const float nw = (p.noise && p.noise_w) ? __ldg(p.noise_w) : 0.f;
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
            const int iy = it.ty * TH + warp, ix = it.tx * TW + g + 8 * hf;
            if (iy >= MH || ix >= MW) continue;
            if constexpr (VOL) {
                int cell, ly, lx;
                if (!vol_cell(p, it.ty, iy, ix, cell, ly, lx)) continue;
                const int b = cell / p.vol.depth, z = cell - b * p.vol.depth;
                const int64_t ro = (((int64_t)b * H + ly) * W + lx) * p.out_ld + z * p.vox_out;
#pragma unroll
                for (int nf = 0; nf < NT / 8; ++nf)
                    epilogue_dense2(p, it.n0 + nf * 8 + 2 * q, acc.d[4 * nf + 2 * hf], acc.d[4 * nf + 2 * hf + 1], ro, p.out + ro);
                continue;
            }
            if constexpr (DENSE) {
                const int64_t ro = (((int64_t)it.b * MH + iy) * MW + ix) * p.out_ld;
                if constexpr (EPI == EPI_SPADE) {
                    const int hs = p.norm_half;
                    const float* xp = p.norm_x + (((int64_t)it.b * (MH >> hs) + (iy >> hs)) * (MW >> hs) + (ix >> hs)) * p.norm_ld;
#pragma unroll
                    for (int nf = 0; nf < NT / 8; ++nf)
                        epilogue_spade(p, it.b, it.n0 + nf * 8 + 2 * q, acc.d[4 * nf + 2 * hf], acc.d[4 * nf + 2 * hf + 1], xp, p.out + ro);
                    continue;
                }
                if constexpr (PW) {
                    const float* up = p.residual_up ? p.residual_up + (((int64_t)it.b * (MH >> 1) + (iy >> 1)) * (MW >> 1) + (ix >> 1)) * p.rup_ld
                                                    : nullptr;
                    const float f = EPI == EPI_FACTOR ? __ldg(p.factor + ((int64_t)it.b * MH + iy) * MW + ix) : 1.f;
#pragma unroll
                    for (int nf = 0; nf < NT / 8; ++nf)
                        epilogue_pw2<EPI == EPI_FACTOR>(p, it.n0 + nf * 8 + 2 * q, acc.d[4 * nf + 2 * hf], acc.d[4 * nf + 2 * hf + 1], ro,
                                                        up, f, p.out + ro);
                    continue;
                }
#pragma unroll
                for (int nf = 0; nf < NT / 8; ++nf)
                    epilogue_dense2(p, it.n0 + nf * 8 + 2 * q, acc.d[4 * nf + 2 * hf], acc.d[4 * nf + 2 * hf + 1], ro, p.out + ro);
                continue;
            }
            const float z = p.noise ? nw * __ldg(p.noise + ((int64_t)(p.noise_b == 1 ? 0 : it.b) * MH + iy) * MW + ix) : 0.f;
            float* dst = p.out + (((int64_t)it.b * MH + iy) * MW + ix) * p.nch;
#pragma unroll
            for (int nf = 0; nf < NT / 8; ++nf) {
                const int n = it.n0 + nf * 8 + 2 * q;
                epilogue2<false>(p, it.b, c[hf], n, z, acc.d[4 * nf + 2 * hf], acc.d[4 * nf + 2 * hf + 1], dst);
            }
        }
    };

    int item = blockIdx.x;
    if (item >= items) return;
    Item cur = decode_item<false>(p, item, NT), nxt;
    int cls[2], cls_n[2];
    float2 sty[2][4], sty_n[2][4];                        // [row][j]: styles of the chunk's fragment channels
    row_classes(cur, cls);                               // DENSE: no label, every row region 0
    if (STY_REG) load_styles(cur, 0, 0, cls, sty);
    int kc = 0, buf = 0;
    // the next (item, chunk): decode it, start its copies into slot buf ^ 1 and load its styles
    auto fetch_next = [&](bool last_chunk, int item_n, int kc_n) {
        if (last_chunk) {
            nxt = decode_item<false>(p, item_n, NT);
            row_classes(nxt, cls_n);
        } else {
            nxt = cur, cls_n[0] = cls[0], cls_n[1] = cls[1];
        }
        prefetch(nxt, kc_n, buf ^ 1);
        if (STY_REG) load_styles(nxt, kc_n, 0, cls_n, sty_n);
    };
    if (RES) copy_block(cur);                            // committed with the first halo
    prefetch(cur, 0, 0);
#pragma unroll 1
    while (true) {
        const bool last_chunk = kc == nchunks - 1;
        const int item_n = last_chunk ? item + (int)gridDim.x : item, kc_n = last_chunk ? 0 : kc + 1;
        const bool more = item_n < items;
        if constexpr (NT == 128) {
            // The chunk's nine taps in TG-tap groups, one weight-ring slot each.  At a
            // group's barrier: its slot is complete and visible to the async proxy, and every thread has retired the MMAs
            // up to the first tap of the previous group (wait_group 1 before building that group's last tap; wait_group 0
            // at the end of a chunk) - so every MMA of the group before that, in both warpgroups.  Its slot, two groups
            // old, is the one refilled, once this group's first MMAs are issued; the previous group's slot may still be
            // read.  The halo slot refilled with the last group was last read by the builds of the previous chunk.
            const uint8_t* halo = smem + buf * stage;
#pragma unroll
            for (int tg = 0; tg < 9 / TG; ++tg) {
                cp_async_wait_all();
                fence_proxy_async();
                __syncthreads();
                const uint32_t bt0 = w_s + ws * W_SLOT;
                ws = ws == 2 ? 0 : ws + 1;                // the slot to refill
#pragma unroll
                for (int k = 0; k < TG; ++k) {
                    const int ti = TG * tg + k, u = ti & 1;
                    if (ti >= 2) wgmma_wait<1>();         // fragment set u: tap ti - 2, its last reader, has retired
                    build(halo, p.taps[ti], sty, fh[u], fl[u]);
                    issue(bt0 + k * B_TAP, fh[u], fl[u], kc == 0 && ti == 0);
                    if (k == 0) {
                        if (tg + 1 < 9 / TG) {
                            copy_group(cur, kc, tg + 1, ws);
                            cp_async_commit();
                        } else if (more) {
                            fetch_next(last_chunk, item_n, kc_n);
                        }
                    }
                }
            }
        } else {
            // slot buf complete and visible to the async proxy; every MMA of the previous chunk retired (wait_group 0 below),
            // so the other slot may be refilled once this chunk's first MMAs are issued
            cp_async_wait_all();
            fence_proxy_async();
            __syncthreads();
            const uint8_t* halo = smem + buf * stage;
            const uint32_t bt0 = RES ? w_s + kc * p.ntaps * B_TAP : smem_s + buf * stage + w_ofs;
            if (STY_SMEM) load_styles(cur, kc, buf, cls, sty);
            build(halo, p.taps[0], sty, fh[0], fl[0]);
            issue(bt0, fh[0], fl[0], kc == 0);
            if (more) fetch_next(last_chunk, item_n, kc_n);      // while the first tap's MMAs run
            // fragment set tap % 2 is rebuilt after wait_group 1 has retired tap - 2, its last reader
    #pragma unroll 1
            for (int ti = 1; ti < p.ntaps; ti += 2) {
                wgmma_wait<1>();
                build(halo, p.taps[ti], sty, fh[1], fl[1]);
                issue(bt0 + ti * B_TAP, fh[1], fl[1], false);
                if (ti + 1 < p.ntaps) {
                    wgmma_wait<1>();
                    build(halo, p.taps[ti + 1], sty, fh[0], fl[0]);
                    issue(bt0 + (ti + 1) * B_TAP, fh[0], fl[0], false);
                }
            }
        }
        wgmma_wait<0>();
        acc.fence();
        if (RES && more && nxt.n0 != cur.n0) {           // next N tile: its block, once both warpgroups' MMAs retired;
            __syncthreads();                              // the barrier at the top of the loop waits for the copies
            copy_block(nxt);
            cp_async_commit();
        }

        if (last_chunk) store_item(cur, cls);
        if (!more) break;
        cur = nxt, item = item_n, kc = kc_n, buf ^= 1;
        cls[0] = cls_n[0], cls[1] = cls_n[1];
        if (STY_REG) {
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int j = 0; j < 4; ++j) sty[h][j] = sty_n[h][j];
        }
    }
}

// ---- 7x7 convolution of every depth slice of a volume (face-vid2vid's dense-motion mask and occlusion, as one GEMM)
// x [B, H, W, D, Cin] -> y [B, D, H, W, 128]: y[b, z, y, x, n] = sum over (ky, kx, c) of w[ky 7 + kx, n, c] x[b, y + ky - 3,
// x + kx - 3, z, c], zero outside the slice; weights [2][49][128][Cin] (bf16 hi, lo).  One CTA per (8 x 16 pixel tile,
// slice): the A operand is built in registers from an fp32 halo tile (conv3x3_rs_kernel's swizzled layout, a 3-pixel
// border: 14 x 22 pixels x 32 channels) and multiplied by the N = 128 weights of one tap with split_mma.  K runs
// chunk-outer, tap-inner: 49 taps of a 32-channel chunk, the chunk's halo loaded once.  The weights stream one tap per
// step through a ring of S7 slots (one cp.async group per step, PD7 = S7 - 2 steps ahead); the next chunk's halo travels
// with the first step of the current chunk, into the other halo slot.  The step invariant is written at the loop.  Every
// output's sum order is fixed by the channel count: bit reproducible and independent of the batch.
constexpr int K7_TAPS = 49, K7_R = 3, K7_HH = TH + 2 * K7_R, K7_HW = TW + 2 * K7_R, K7_HPIX = K7_HH * K7_HW;
constexpr int K7_HALO = K7_HPIX * KC * 4;               // 39424
constexpr int K7_NT = 128, K7_BPLANE = K7_NT * KC * 2, K7_BTAP = 2 * K7_BPLANE;
constexpr int S7 = 8, PD7 = S7 - 2;
constexpr size_t K7_SMEM = 128 + 2 * (size_t)K7_HALO + (size_t)S7 * K7_BTAP;

template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__global__ void __launch_bounds__(NUM_THREADS, 1)
    conv7x7_slices_kernel(const float* __restrict__ x, const __nv_bfloat16* __restrict__ wt, float* __restrict__ y, int depth,
                          int h, int w, int cin, int tiles_x) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~uintptr_t(127));
    const uint32_t smem_s = (uint32_t)__cvta_generic_to_shared(smem);
    const uint32_t w_s = smem_s + 2 * K7_HALO;
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5, g = lane >> 2, q = lane & 3, hc = t & 7;
    const int tx = blockIdx.x % tiles_x, ty = blockIdx.x / tiles_x, z = blockIdx.y, b = blockIdx.z;
    const int nsteps = (cin / KC) * K7_TAPS;
    const int64_t vp = (int64_t)depth * cin;              // pixel pitch of x

    // halo slot kc & 1 <- chunk kc of the tile's 14 x 22 pixels of slice z, zero outside the slice
    auto copy_halo = [&](int kc) {
        const uint32_t st = smem_s + (kc & 1) * K7_HALO;
        const float* xb = x + ((int64_t)b * h * w) * vp + (int64_t)z * cin + kc * KC + hc * 4;
        for (int hp = t >> 3; hp < K7_HPIX; hp += NUM_THREADS / 8) {
            const int hy = hp / K7_HW, sy = ty * TH - K7_R + hy, sx = tx * TW - K7_R + hp - hy * K7_HW;
            const bool ok = sy >= 0 && sy < h && sx >= 0 && sx < w;
            cp_async16(st + hp * 128 + ((hc ^ (hp & 7)) << 4), ok ? xb + ((int64_t)sy * w + sx) * vp : x, ok ? 16 : 0);
        }
    };
    // weight slot s % S7 <- tap s % 49 of chunk s / 49, both planes in the no-swizzle K-major core-matrix layout (copy c
    // of a plane: row 8 (c / 32) + c % 8, channel quad (c / 8) % 4, at byte 16 c)
    auto copy_tap = [&](int s) {
        const int kc = s / K7_TAPS, tap = s - kc * K7_TAPS;
        const uint32_t dst = w_s + (s % S7) * K7_BTAP;
#pragma unroll
        for (int i = 0; i < 2 * K7_BPLANE / 16 / NUM_THREADS; ++i) {
            const int e = t + NUM_THREADS * i, hl = e / (K7_BPLANE / 16), c = e % (K7_BPLANE / 16);
            const int n = (c >> 5) * 8 + (c & 7);
            cp_async16(dst + hl * K7_BPLANE + c * 16,
                       wt + ((int64_t)(hl * K7_TAPS + tap) * K7_NT + n) * cin + kc * KC + ((c >> 3) & 3) * 8, 16);
        }
    };

    SplitAcc<K7_NT> acc{};                                // zero: the fences read every register
    uint32_t fh[2][2][4], fl[2][2][4];                    // [step % 2][K16 slice][register]: x_hi, x_lo fragments
    // fragment register r of slice ks: row g + 8 (r & 1) of tile row `warp`, channels 16 ks + 8 (r >> 1) + 2 q, + 1
    auto build = [&](const uint8_t* halo, int tap, uint32_t (&hi)[2][4], uint32_t (&lo)[2][4]) {
        const int dy = tap / 7, dx = tap % 7;
#pragma unroll
        for (int ks = 0; ks < 2; ++ks)
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                const int j = 2 * ks + (r >> 1);
                const int hp = (warp + dy) * K7_HW + g + 8 * (r & 1) + dx;
                const float2 v = *reinterpret_cast<const float2*>(halo + hp * 128 + (((2 * j + (q >> 1)) ^ (hp & 7)) << 4) + (q & 1) * 8);
                split2(v.x, v.y, hi[ks][r], lo[ks][r]);
            }
    };

    copy_halo(0);
    for (int s = 0; s < PD7; ++s) {                       // one group per step: step 0 carries chunk 0's halo
        if (s < nsteps) copy_tap(s);
        cp_async_commit();
    }
#pragma unroll 1
    for (int s = 0; s < nsteps; ++s) {
        // Step s: groups 0 .. s + PD7 - 1 are committed, so waiting for all but the newest PD7 - 1 completes group s (its
        // weights and, at a chunk's first step, the halo issued one chunk earlier).  Past the barrier every thread has
        // retired the MMAs of step s - 2 (wait_group 1 after issuing step s - 1): its fragment set (s & 1) and weight
        // slot ((s + PD7) % S7) are free.  The other halo slot was last read by the builds of the previous chunk.
        cp_async_wait<PD7 - 1>();
        fence_proxy_async();
        __syncthreads();
        const int kc = s / K7_TAPS, tap = s - kc * K7_TAPS, u = s & 1;
        build(smem + (kc & 1) * K7_HALO, tap, fh[u], fl[u]);
        acc.fence();
        fence_frag(fh[u]);
        fence_frag(fl[u]);
        wgmma_fence();
        const uint32_t bt = w_s + (s % S7) * K7_BTAP;
#pragma unroll
        for (int ks = 0; ks < 2; ++ks)
            split_mma(acc, fh[u][ks], fl[u][ks], bt + ks * 2 * LBO, bt + ks * 2 * LBO + K7_BPLANE, (s == 0 && ks == 0) ? 0 : 1);
        wgmma_commit();
        acc.fence();
        fence_frag(fh[u]);
        fence_frag(fl[u]);
        if (tap == 0 && (kc + 1) * K7_TAPS < nsteps) copy_halo(kc + 1);
        if (s + PD7 < nsteps) copy_tap(s + PD7);
        cp_async_commit();
        wgmma_wait<1>();
    }
    wgmma_wait<0>();
    acc.fence();
    acc.fold();
    // this thread's rows g, g + 8 of tile row `warp`; register 4 nf + 2 hf + e: column 8 nf + 2 q + e
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) {
        const int iy = ty * TH + warp, ix = tx * TW + g + 8 * hf;
        float* dst = y + ((((int64_t)b * depth + z) * h + iy) * w + ix) * K7_NT + 2 * q;
#pragma unroll
        for (int nf = 0; nf < K7_NT / 8; ++nf)
            *reinterpret_cast<float2*>(dst + nf * 8) = make_float2(acc.d[4 * nf + 2 * hf], acc.d[4 * nf + 2 * hf + 1]);
    }
}

// ------------------------------------------------------------------------------------------ host
static int num_sms() { return e4s_num_sms(); }

// N-tile width (output channels per work item): 64 when the channel count allows it and the launch still has work for
// half the SMs, else 32.  E4S_B200_NTILE=32|64 forces a width the channel count allows.
static int pick_ntile(int channels, int64_t items_per_ntile_column) {
    if (const char* f = getenv("E4S_B200_NTILE")) {
        const int v = atoi(f);
        if ((v == 32 || v == 64) && channels % v == 0) return v;
    }
    if (channels % 64 != 0) return 32;
    return items_per_ntile_column * (channels / 64) >= num_sms() / 2 ? 64 : 32;
}

// Gradient work items: a (pixel tile, N tile) pair is a serial chain of (regions in the tile) x parity planes x taps x
// Cout / 32 K steps.  The low-resolution layers of one face have a handful of pairs with every region in each: when the
// pairs cannot fill the SMs, cut the chain - region passes first (up to ncls ways), then parity planes; the partial sums
// meet in gx through atomics (gx zeroed first) and in gs through the atomics the kernel uses anyway.
// E4S_B200_DGRAD_SPLIT="G,H" forces a split (tests).
static void choose_split(int64_t pairs, int ncls, int nph, int& gsplit, int& hsplit) {
    gsplit = hsplit = 1;
    if (const char* f = getenv("E4S_B200_DGRAD_SPLIT")) {
        int g = 0, h = 0;
        if (sscanf(f, "%d,%d", &g, &h) == 2 && g >= 1 && (h == 1 || h == 2 || h == 4)) {
            gsplit = g < ncls ? g : ncls, hsplit = h < nph ? h : nph;
            return;
        }
    }
    const int sms = num_sms();
    if (pairs >= 2 * sms) return;
    // aim at ~4 work items per SM: the chains differ in length (regions per tile)
    const int64_t g = e4s_ceil_div(4 * sms, pairs);
    gsplit = (int)(g < ncls ? g : ncls);
    while (hsplit < nph && pairs * gsplit * hsplit < sms) hsplit *= 2;
}

static void set_taps(Params& p, int tap_mask) {
    p.ntaps = 0;
    for (int t = 0; t < 9; ++t)
        if (!tap_mask || ((tap_mask >> t) & 1)) p.taps[p.ntaps++] = t;
}

template <int NT, int MODE>
static int launch_nt(Params p, int64_t outer, cudaStream_t st) {
    p.n_tiles = p.nch / NT;
    const int64_t items = (int64_t)p.tiles_x * p.tiles_y * p.batch * p.n_tiles * outer;
    static E4sSmemOptIn optin;
    if constexpr (MODE == FWD_RS || MODE == FWD_DENSE || MODE == FWD_REFL || MODE == FWD_PW || MODE == FWD_VOL ||
                  MODE == FWD_SPADE || MODE == FWD_PWF) {
        constexpr bool REFL = MODE == FWD_REFL, PW = MODE == FWD_PW || MODE == FWD_PWF, VOL = MODE == FWD_VOL;
        constexpr bool DENSE = MODE == FWD_DENSE || REFL || PW || VOL || MODE == FWD_SPADE;
        constexpr int EPI = MODE == FWD_SPADE ? EPI_SPADE : MODE == FWD_PWF ? EPI_FACTOR : EPI_PLAIN;
        // persistent, as many CTAs per SM as fit (the two ring slots of a 64-channel tile with nine streamed taps take
        // 189 KB of shared memory)
        const int64_t ld = DENSE ? (p.a_ld > p.out_ld ? p.a_ld : p.out_ld) : p.kch;
        if (items >= (1ll << 31) - 1024 || (int64_t)p.h * p.w * ld >= (1ll << 31) || 18ll * p.nch * p.kch >= (1ll << 31))
            return E4S_ERR_SHAPE;
        // the weights stay resident when the N tile's whole block fits beside the two ring slots (halo and styles);
        // E4S_B200_RS_STREAM=1 streams them with every chunk regardless (tests)
        // (PW: the "taps" are the K chunks of a slot, the block is every chunk once, the halo the slot's pixel tiles)
        const int64_t tap_bytes = 2 * NT * KC * 2, block = (int64_t)(p.kch / KC) * (PW ? 1 : p.ntaps) * tap_bytes;
        const int halo = PW ? p.ntaps * M * KC * 4 : HALO_BYTES;
        const int res_slot = halo + (NT == 32 && !DENSE ? p.ncls * KC * 4 : 0);   // resident ring slot: halo (, styles)
        const char* f = getenv("E4S_B200_RS_STREAM");
        // N = 128: never resident; the two slots hold halos, and a ring of three 3-tap weight slots follows them (190 KB)
        constexpr bool WIDE = NT == 128;
        if (WIDE && p.ntaps != 9) return E4S_ERR_SHAPE;
        const bool resident = !WIDE && !(f && atoi(f) != 0) && 128 + 2 * res_slot + block <= e4s_smem_optin_limit();
        const int stage = resident || WIDE ? res_slot : halo + p.ntaps * (int)tap_bytes;
        const size_t smem = 128 + 2 * (size_t)stage + (resident ? (size_t)block : WIDE ? 9 * (size_t)tap_bytes : 0);
        static E4sSmemOptIn optin_res;
        static E4sOccupancy occ[2];
        auto kernel = conv3x3_rs_kernel<NT, false, DENSE, REFL, PW, VOL, false, EPI>;
        if constexpr (!WIDE)
            if (resident) kernel = conv3x3_rs_kernel<NT, true, DENSE, REFL, PW, VOL, false, EPI>;
        if (const int rc = e4s_smem_optin(resident ? optin_res : optin, kernel, smem)) return rc;
        const int per_sm = e4s_ctas_per_sm(occ[resident], kernel, NUM_THREADS, smem);
        const int64_t slots = (int64_t)num_sms() * (per_sm > 1 ? per_sm : 1);
        const int64_t grid = items < slots ? items : slots;
        kernel<<<(unsigned)grid, NUM_THREADS, smem, st>>>(p, (int)items, stage);
    } else {
        if (items >= (1ll << 31)) return E4S_ERR_SHAPE;
        constexpr size_t smem = 1024 + (size_t)NSTAGE * (2 * A_PLANE + 2 * NT * KC * 2);
        if (const int rc = e4s_smem_optin(optin, conv3x3_wgmma_kernel<NT, MODE>, smem)) return rc;
        conv3x3_wgmma_kernel<NT, MODE><<<(unsigned)items, NUM_THREADS, smem, st>>>(p);
    }
    return e4s_launch_status();
}

// nt: channels per work item (pick_ntile)
template <int MODE>
static int launch(const Params& p, int nt, int64_t outer, cudaStream_t st) {
    if (nt == 32) return launch_nt<32, MODE>(p, outer, st);
    if constexpr (MODE == FWD_RS)
        if (nt == 128) return launch_nt<128, MODE>(p, outer, st);
    return launch_nt<64, MODE>(p, outer, st);
}

// pixel tiles over the output row grid (the input grid unless the caller set another one)
static void tiles(Params& p) {
    if (!p.mh) p.mh = p.h, p.mw = p.w;
    p.tiles_x = (int)e4s_ceil_div(p.mw, TW);
    p.tiles_y = (int)e4s_ceil_div(p.mh, TH);
}

template <int MODE = FWD>
static int forward(Params p, cudaStream_t st) {
    tiles(p);
    const int64_t pixel_tiles = (int64_t)p.tiles_x * p.tiles_y * p.batch;
    // up-sampling layer: one output parity per work item, or all four in one item once the items already fill the GPU
    // twice over without the split (four times fewer operand-ring fills); E4S_B200_UP2=1 | 0 forces either (tests)
    const int nt = pick_ntile(p.nch, pixel_tiles * (p.up ? 4 : 1));
    p.parity_items = pixel_tiles * (p.nch / nt) < 2 * num_sms();
    if (const char* f = getenv("E4S_B200_UP2")) p.parity_items = atoi(f) != 0;
    const int64_t outer = (p.up && p.parity_items) ? 4 : 1;
    return launch<MODE>(p, nt, outer, st);
}

// N-tile width of the plain modulated layers on the register-operand kernel: 128 when the channel count allows it and
// the 64-channel items would not fit in one wave of CTAs (one per SM), else pick_ntile's choice.  A 128-channel item
// takes ~1.5x the time of a 64-channel one (0.186 against 0.124 ms at 512 -> 512 channels): 1.27 - 1.33x faster where
// both widths run several waves or 128 saves one of two, 0.67x where 64 already ran in one (H100 80GB HBM3, 700 W;
// DESIGN.md section 9).  E4S_B200_RS_NTILE=64|128 forces a width the channel count allows; a set E4S_B200_NTILE keeps
// pick_ntile's choice.
static int pick_ntile_rs(int channels, int64_t pixel_tiles) {
    const char* f = getenv("E4S_B200_RS_NTILE");
    const int v = f ? atoi(f) : 0;
    if ((v == 64 || v == 128) && channels % v == 0) return v;
    if (channels % 128 == 0 && !getenv("E4S_B200_NTILE") && 2 * pixel_tiles * (channels / 128) > num_sms()) return 128;
    return pick_ntile(channels, pixel_tiles);
}

// plain modulated convolution (p.up == 0, p.out_stride == 1, no shift): the register-operand kernel
static int forward_rs(Params p, cudaStream_t st) {
    tiles(p);
    const int nt = pick_ntile_rs(p.nch, (int64_t)p.tiles_x * p.tiles_y * p.batch);
    return launch<FWD_RS>(p, nt, 1, st);
}

// The unmasked transposed-convolution GEMM (conv3x3_rs_kernel's CONVT mode), persistent, one CTA per SM.
static int launch_convt(const Params& p, int64_t items, cudaStream_t st) {
    if (items >= (1ll << 31) - 1024 || (int64_t)p.h * p.w * p.kch >= (1ll << 31) || 18ll * p.nch * p.kch >= (1ll << 31))
        return E4S_ERR_SHAPE;
    // the weights stay resident when every chunk's class tiles fit beside the two halo slots; E4S_B200_RS_STREAM=1
    // streams them with every chunk regardless (tests)
    const int halo = CT_HPIX * KC * 4;
    const int64_t block = (int64_t)(p.kch / KC) * CT_CHUNK;
    const char* f = getenv("E4S_B200_RS_STREAM");
    const bool resident = !(f && atoi(f) != 0) && 128 + 2 * halo + block <= e4s_smem_optin_limit();
    const int stage = resident ? halo : halo + CT_CHUNK;
    const size_t smem = 128 + 2 * (size_t)stage + (resident ? (size_t)block : 0);
    static E4sSmemOptIn optin[2];
    auto kernel = resident ? conv3x3_rs_kernel<128, true, false, false, false, false, true>
                           : conv3x3_rs_kernel<128, false, false, false, false, false, true>;
    if (const int rc = e4s_smem_optin(optin[resident], kernel, smem)) return rc;
    const int64_t grid = items < num_sms() ? items : num_sms();
    kernel<<<(unsigned)grid, NUM_THREADS, smem, st>>>(p, (int)items, stage);
    return e4s_launch_status();
}

// N-tile width of the gathered-row GEMM (one class of Cout channels per item): 128 when Cout allows it and the items at
// that width (row blocks x 4 classes x Cout / 128, counted to the cap) fill the SMs twice, else 64 where Cout allows it,
// else 32.  64 and 128 give the same bits; the stacked 32-channel form is taken only where 64 does not divide Cout, so the
// width never changes a result.  E4S_B200_RS_NTILE=64|128 forces a width Cout allows (tests).
static int pick_ntile_rows(int cout, int64_t row_blocks) {
    const char* f = getenv("E4S_B200_RS_NTILE");
    const int v = f ? atoi(f) : 0;
    if ((v == 64 || v == 128) && cout % v == 0) return v;
    if (cout % 128 == 0 && row_blocks * 4 * (cout / 128) >= 2 * num_sms()) return 128;
    return cout % 64 == 0 ? 64 : 32;
}

// The masked transposed-convolution GEMM (conv3x3_rs_kernel's ROWS mode), persistent: p.tiles_x row blocks per sample,
// p.n_tiles = Cout / nt slices per class.  A ring slot holds up to four K steps (p.ntaps), as many as two slots fit.
template <int NT>
static int launch_rows(Params p, cudaStream_t st) {
    p.n_tiles = p.nch / 4 / NT;
    const int64_t items = (int64_t)p.tiles_x * p.batch * 4 * p.n_tiles;
    if (items >= (1ll << 31) - 1024 || (int64_t)p.h * p.w * p.kch >= (1ll << 31) || 18ll * p.nch * p.kch >= (1ll << 31))
        return E4S_ERR_SHAPE;
    // p.ntaps: K steps per ring slot (this mode has no tap list; the taps follow the class), as many as two slots fit
    const int step = M * KC * 4 + 2 * NT * KC * 2;        // gathered rows + both weight planes
    p.ntaps = (e4s_smem_optin_limit() - 128) / (2 * step);
    if (p.ntaps > 4) p.ntaps = 4;
    if (p.ntaps < 1) return E4S_ERR_SHAPE;
    const int stage = p.ntaps * step;
    const size_t smem = 128 + 2 * (size_t)stage;
    static E4sSmemOptIn optin;
    auto kernel = conv3x3_rs_kernel<NT, false, false, false, false, false, false, EPI_PLAIN, true>;
    if (const int rc = e4s_smem_optin(optin, kernel, smem)) return rc;
    const int64_t grid = items < num_sms() ? items : num_sms();
    kernel<<<(unsigned)grid, NUM_THREADS, smem, st>>>(p, (int)items, stage);
    return e4s_launch_status();
}

// ---- unmasked up-sampling layer: transposed-convolution GEMM + blur pass
// The stride-2 transposed convolution u[p] = sum_i x[i] w[p - 2 i] (per axis) is stored space-to-depth on a row grid one
// pixel larger than the input: T'[m, n, (a, c), o] = u[2m + a, 2n + c, o] for m <= H, n <= W.  Along an axis, parity a = 0
// takes the taps d = 0 (weight row 2) and d = 1 (row 0) of the source rows m - 1 + d, parity a = 1 only d = 1 (row 1).  So
// it is a stride-1 convolution over the 2 x 2 taps {0, 1, 3, 4} with N = 4 Cout class-stacked channels, and class (a, c)
// uses 4, 2, 2 or 1 of those taps: 9 tap products per input pixel, all four classes in one work item of
// conv3x3_rs_kernel's CONVT mode.  The gathered-row GEMM of the masked layers (its ROWS mode) has one class per work item
// instead, over that class's own taps.

constexpr int BLUR_ROWS = 32;                         // output rows per thread of the blur pass
constexpr int BLUR_THREADS = 256;

// y[Y, X, o] = act(demod[o] * sum_{p,q} fir[3-p][3-q] T[Y-1+p][X-1+q] + noise_w * noise[Y, X] + bias[o]), the true 4 x 4
// convolution (pad 1) of T = the transposed-convolution output, T[u, v] = T'[u >> 1, v >> 1, (u & 1, v & 1)], zero
// outside 0 <= u <= 2H + 1.  A thread owns 4 channels of the output columns 2j, 2j + 1 over BLUR_ROWS rows and walks down
// T one row at a time: the row's five float4 (T columns 2j - 1 .. 2j + 3) feed the four output rows it touches, and the
// row it completes is stored.  Every output sums p = 0..3, q = 0..3 in that order: the result does not depend on the
// thread layout.
__global__ void __launch_bounds__(BLUR_THREADS, 3) convt_blur_kernel(const float* __restrict__ t, const float* __restrict__ fir,
                                                                  const float* __restrict__ demod,
                                                                  const float* __restrict__ noise,
                                                                  const float* __restrict__ noise_w,
                                                                  const float* __restrict__ bias, float* __restrict__ y,
                                                                  int batch, int h, int w, int cout, int noise_b, int act,
                                                                  int strips) {
    const int cq = cout >> 2;
    int64_t gid = (int64_t)blockIdx.x * BLUR_THREADS + threadIdx.x;
    if (gid >= (int64_t)batch * strips * w * cq) return;
    const int o = (int)(gid % cq) * 4;
    gid /= cq;
    const int j = (int)(gid % w);
    gid /= w;
    const int y0 = (int)(gid % strips) * BLUR_ROWS, b = (int)(gid / strips);
    const int Ho = 2 * h, Wo = 2 * w;
    float f[4][4];
#pragma unroll
    for (int q = 0; q < 16; ++q) f[q >> 2][q & 3] = __ldg(fir + 15 - q);
    const float4 d = demod ? ld4(demod + (int64_t)b * cout + o) : make_float4(1.f, 1.f, 1.f, 1.f);
    const float4 bv = bias ? ld4(bias + o) : make_float4(0.f, 0.f, 0.f, 0.f);
    const float nw = (noise && noise_w) ? __ldg(noise_w) : 0.f;
    const int64_t trow = (int64_t)(w + 1) * 4 * cout;                   // floats per T' row
    const float* tb = t + (int64_t)b * (h + 1) * trow + o;
    // acc[i]: output row Y = u - 2 + i, which T row u reaches through FIR row p = 3 - i
    float4 acc[4][2];
#pragma unroll
    for (int i = 0; i < 4; ++i) acc[i][0] = acc[i][1] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 4
    for (int r = 0; r < BLUR_ROWS + 3; ++r) {
        const int u = y0 - 1 + r;
        float4 v[5];
#pragma unroll
        for (int k = 0; k < 5; ++k) v[k] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (u >= 0 && (u >> 1) <= h) {
            // T column 2j - 1 + k: T' pixel j + ((k - 1) >> 1), class column (k + 1) & 1
            const float* row = tb + (int64_t)(u >> 1) * trow + (int64_t)((u & 1) * 2) * cout + (int64_t)j * 4 * cout;
            if (j > 0) v[0] = ld4(row - 3 * cout);
            v[1] = ld4(row);
            v[2] = ld4(row + cout);
            v[3] = ld4(row + 4 * cout);
            v[4] = ld4(row + 5 * cout);
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int p = 3 - i;
#pragma unroll
            for (int cx = 0; cx < 2; ++cx) {
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const float c = f[p][q];
                    const float4 e = v[cx + q];
                    float4& a = acc[i][cx];
                    a.x = fmaf(c, e.x, a.x), a.y = fmaf(c, e.y, a.y), a.z = fmaf(c, e.z, a.z), a.w = fmaf(c, e.w, a.w);
                }
            }
        }
        const int yo = u - 2;                         // complete: its p = 3 row was this one
        if (r >= 3 && yo < Ho) {
#pragma unroll
            for (int cx = 0; cx < 2; ++cx) {
                const int xo = 2 * j + cx;
                const float z = noise ? nw * __ldg(noise + ((int64_t)(noise_b == 1 ? 0 : b) * Ho + yo) * Wo + xo) : 0.f;
                *reinterpret_cast<float4*>(y + (((int64_t)b * Ho + yo) * Wo + xo) * cout + o) = epilogue4(acc[0][cx], d, z, bv, act);
            }
        }
#pragma unroll
        for (int i = 0; i < 3; ++i) acc[i][0] = acc[i + 1][0], acc[i][1] = acc[i + 1][1];
        acc[3][0] = acc[3][1] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
}

// ---- masked up-sampling layer: transposed-convolution GEMM over (T' pixel, region) rows + region-aware blur pass
// Through the 4 x 4 blur, T' pixel (m, n) (T rows 2m, 2m + 1) reaches only the output pixels Y in [2m - 2, 2m + 2],
// X in [2n - 2, 2n + 2].  It is computed once with the style of each region present in that (clipped) window and for no
// other region; an output pixel of region r reads the rows of its own region, which its window always holds.

constexpr int LIST_THREADS = 1024;
constexpr int BLUR_PIX = 4;                           // output pixels per thread of the masked blur pass

// One block per sample.  need[b, m, n]: the regions of the 5 x 5 window; base[b, m, n]: exclusive prefix sum of their
// counts in row-major (m, n) order; rows[b, base + k]: (m, n, k-th region of need) for rows below cap; count[b]: the
// sample's total (the list is complete only when count <= cap; past cap, count is only known to exceed it).
__global__ void __launch_bounds__(LIST_THREADS) convt_row_list_kernel(const uint8_t* __restrict__ label, uint32_t* __restrict__ need,
                                                                      int* __restrict__ base, int* __restrict__ count,
                                                                      uint32_t* __restrict__ rows, int h, int w, int ncls, int cap) {
    __shared__ int warp_sum[LIST_THREADS / 32];
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5, b = blockIdx.x;
    const int Ho = 2 * h, Wo = 2 * w, npix = (h + 1) * (w + 1);
    const uint8_t* lb = label + (int64_t)b * Ho * Wo;
    int running = 0;
    for (int start = 0; start < npix; start += LIST_THREADS) {
        const int pix = start + t, m = pix / (w + 1), n = pix % (w + 1);
        uint32_t bits = 0;
        if (pix < npix) {
            for (int Y = max(2 * m - 2, 0); Y <= min(2 * m + 2, Ho - 1); ++Y)
                for (int X = max(2 * n - 2, 0); X <= min(2 * n + 2, Wo - 1); ++X)
                    bits |= 1u << region(lb, ncls, Y * Wo + X);
        }
        const int c = __popc(bits);
        int incl = c;                                 // block-wide inclusive scan: within the warp, then over warps
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int v = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += v;
        }
        if (lane == 31) warp_sum[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            int s = warp_sum[lane];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int v = __shfl_up_sync(0xffffffffu, s, o);
                if (lane >= o) s += v;
            }
            warp_sum[lane] = s;
        }
        __syncthreads();
        const int excl = running + (warp ? warp_sum[warp - 1] : 0) + incl - c;
        if (pix < npix) {
            const int64_t gp = (int64_t)b * npix + pix;
            need[gp] = bits;
            base[gp] = excl;
            int i = excl;
            for (uint32_t rb = bits; rb && i < cap; rb &= rb - 1, ++i) rows[(int64_t)b * cap + i] = row_pack(m, n, __ffs(rb) - 1);
        }
        running += warp_sum[LIST_THREADS / 32 - 1];
        __syncthreads();                              // warp_sum is rewritten by the next chunk
        if (running > cap) break;                     // the sample falls back: its list is not read
    }
    if (t == 0) count[b] = running;
}

// y[Y, X, o] = act(demod[r, o] * sum_{p,q} fir[3-p][3-q] T_r[Y-1+p][X-1+q] + noise_w * noise[Y, X] + bias[o]) with
// r = label[Y, X] and T_r the transposed-convolution output computed with region r's style: T_r[u, v] is channel
// ((u & 1, v & 1), o) of compacted row base[m, n] + popcount(need[m, n] & ((1 << r) - 1)), (m, n) = (u >> 1, v >> 1); zero
// for u < 0 or v < 0.  A thread owns 4 channels of BLUR_PIX output pixels along X; p = 0..3, q = 0..3 are summed in that
// order.
// Samples whose list overflowed (count > cap) are left to the folded kernel.
__global__ void __launch_bounds__(BLUR_THREADS) convt_blur_masked_kernel(
    const float* __restrict__ tc, const uint32_t* __restrict__ need, const int* __restrict__ base, const int* __restrict__ count,
    const uint8_t* __restrict__ label, const float* __restrict__ fir, const float* __restrict__ demod,
    const float* __restrict__ noise, const float* __restrict__ noise_w, const float* __restrict__ bias, float* __restrict__ y,
    int batch, int h, int w, int cout, int ncls, int cap, int noise_b, int act) {
    const int cq = cout >> 2, Ho = 2 * h, Wo = 2 * w, xg = (Wo + BLUR_PIX - 1) / BLUR_PIX;
    int64_t gid = (int64_t)blockIdx.x * BLUR_THREADS + threadIdx.x;
    if (gid >= (int64_t)batch * Ho * xg * cq) return;
    const int o = (int)(gid % cq) * 4;
    gid /= cq;
    const int X0 = (int)(gid % xg) * BLUR_PIX;
    gid /= xg;
    const int Y = (int)(gid % Ho), b = (int)(gid / Ho);
    if (__ldg(count + b) > cap) return;
#pragma unroll 1
    for (int X = X0; X < min(X0 + BLUR_PIX, Wo); ++X) {
        const int r = region(label, ncls, ((int64_t)b * Ho + Y) * Wo + X);
        const uint32_t below = (1u << r) - 1u;
        const int64_t pix0 = (int64_t)b * (h + 1) * (w + 1);
        const float* tb = tc + (int64_t)b * cap * 4 * cout + o;
        // T rows Y - 1 .. Y + 2 lie in T' rows m0 + (p + ey) / 2 (2 of them for odd Y, 3 for even Y); the same along x.  All
        // lookups, then all loads, are issued before the first is used.
        const int m0 = (Y - 1) >> 1, n0 = (X - 1) >> 1, ey = 1 - (Y & 1), ex = 1 - (X & 1);
        int rowi[3][3];
#pragma unroll
        for (int i = 0; i < 3; ++i)
#pragma unroll
            for (int j = 0; j < 3; ++j) {
                const int64_t pi = pix0 + (int64_t)min(max(m0 + i, 0), h) * (w + 1) + min(max(n0 + j, 0), w);
                rowi[i][j] = __ldg(base + pi) + __popc(__ldg(need + pi) & below);
            }
        float4 e[4][4];
#pragma unroll
        for (int p = 0; p < 4; ++p)
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int u = Y - 1 + p, v = X - 1 + q;
                const int ra = ey ? (ex ? rowi[(p + 1) >> 1][(q + 1) >> 1] : rowi[(p + 1) >> 1][q >> 1])
                                  : (ex ? rowi[p >> 1][(q + 1) >> 1] : rowi[p >> 1][q >> 1]);
                e[p][q] = make_float4(0.f, 0.f, 0.f, 0.f);
                if (u >= 0 && v >= 0) e[p][q] = ld4(tb + ((int64_t)ra * 4 + (u & 1) * 2 + (v & 1)) * cout);
            }
        float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int p = 0; p < 4; ++p)
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const float c = __ldg(fir + 15 - 4 * p - q);
                a.x = fmaf(c, e[p][q].x, a.x), a.y = fmaf(c, e[p][q].y, a.y), a.z = fmaf(c, e[p][q].z, a.z), a.w = fmaf(c, e[p][q].w, a.w);
            }
        const float4 d = demod ? ld4(demod + ((int64_t)b * ncls + r) * cout + o) : make_float4(1.f, 1.f, 1.f, 1.f);
        const float4 bv = bias ? ld4(bias + o) : make_float4(0.f, 0.f, 0.f, 0.f);
        const float z = noise ? __ldg(noise_w) * __ldg(noise + ((int64_t)(noise_b == 1 ? 0 : b) * Ho + Y) * Wo + X) : 0.f;
        *reinterpret_cast<float4*>(y + (((int64_t)b * Ho + Y) * Wo + X) * cout + o) = epilogue4(a, d, z, bv, act);
    }
}

// Argument checks of the modulated forward entries; the first failing one gives the error code.  ok_shape: the entry's
// own shape limits.
static int check_modconv_fwd(const float* x, const void* w_hilo, const float* s, const float* demod, const uint8_t* label,
                             const float* noise, const float* noise_w, const float* bias, const float* y, int batch, int h,
                             int w, int cin, int cout, int ncls, int noise_b, bool ok_shape) {
    E4S_REQUIRE(x && w_hilo && s && y, E4S_ERR_ARG);
    E4S_REQUIRE(batch > 0 && h > 0 && w > 0 && cin > 0 && cout > 0 && ncls > 0 && ncls <= 32, E4S_ERR_ARG);
    E4S_REQUIRE((cin % 32) == 0 && (cout % 32) == 0 && ok_shape, E4S_ERR_SHAPE);
    E4S_REQUIRE(label || ncls == 1, E4S_ERR_ARG);
    E4S_REQUIRE(!noise || (noise_w && (noise_b == 1 || noise_b == batch)), E4S_ERR_ARG);
    E4S_REQUIRE(e4s_aligned16(x) && e4s_aligned16(w_hilo) && e4s_aligned16(s) && e4s_aligned16(y) &&
                    (!demod || e4s_aligned16(demod)) && (!bias || e4s_aligned16(bias)),
                E4S_ERR_ALIGN);
    return E4S_OK;
}

}  // namespace wgmma_conv

extern "C" int e4s_modconv3x3_tcr_fwd(const float* x, const void* w_hilo_bf16, const float* s, const float* demod,
                                      const uint8_t* label, const float* noise, const float* noise_w, const float* bias,
                                      float* y, int batch, int h, int w, int cin, int cout, int ncls, int up, int noise_b,
                                      int act, void* stream) {
    if (const int rc = wgmma_conv::check_modconv_fwd(x, w_hilo_bf16, s, demod, label, noise, noise_w, bias, y, batch, h, w,
                                                     cin, cout, ncls, noise_b, true))
        return rc;
    wgmma_conv::Params p{};
    p.a = x, p.wt = static_cast<const __nv_bfloat16*>(w_hilo_bf16), p.s = s, p.demod = demod, p.label = label;
    p.noise = noise, p.noise_w = noise_w, p.bias = bias, p.out = y;
    p.batch = batch, p.h = h, p.w = w, p.kch = cin, p.nch = cout, p.ncls = ncls, p.noise_b = noise_b, p.act = act ? 1 : 0;
    p.up = up ? 1 : 0;
    wgmma_conv::set_taps(p, 0);
    return up ? wgmma_conv::forward(p, (cudaStream_t)stream) : wgmma_conv::forward_rs(p, (cudaStream_t)stream);
}

// Host-only: the N-tile width forward_rs picks for this shape (see pick_ntile_rs); no launch, no device access beyond the
// SM count.
extern "C" int e4s_modconv3x3_tcr_fwd_plan(int batch, int h, int w, int cout, int* ntile) {
    E4S_REQUIRE(ntile && batch > 0 && h > 0 && w > 0 && cout > 0, E4S_ERR_ARG);
    E4S_REQUIRE((cout % 32) == 0, E4S_ERR_SHAPE);
    *ntile = wgmma_conv::pick_ntile_rs(cout, e4s_ceil_div(w, wgmma_conv::TW) * e4s_ceil_div(h, wgmma_conv::TH) * batch);
    return E4S_OK;
}

extern "C" int e4s_modconv3x3_up_tcr_fwd(const float* x, const void* wt_hilo_bf16, const float* fir4x4, const float* s,
                                         const float* demod, const float* noise, const float* noise_w, const float* bias,
                                         float* t_buf, float* y, int batch, int h, int w, int cin, int cout, int noise_b,
                                         int act, void* stream) {
    namespace wc = wgmma_conv;
    E4S_REQUIRE(fir4x4 && t_buf, E4S_ERR_ARG);
    if (const int rc = wc::check_modconv_fwd(x, wt_hilo_bf16, s, demod, nullptr, noise, noise_w, bias, y, batch, h, w, cin,
                                             cout, 1, noise_b, true))
        return rc;
    E4S_REQUIRE(e4s_aligned16(t_buf), E4S_ERR_ALIGN);
    cudaStream_t st = (cudaStream_t)stream;
    wc::Params p{};
    p.a = x, p.wt = static_cast<const __nv_bfloat16*>(wt_hilo_bf16), p.s = s, p.out = t_buf;
    p.batch = batch, p.h = h, p.w = w, p.mh = h + 1, p.mw = w + 1, p.kch = cin, p.nch = 4 * cout, p.ncls = 1;
    wc::tiles(p);
    if (const int rc = wc::launch_convt(p, (int64_t)p.tiles_x * p.tiles_y * batch * (cout / 32), st)) return rc;
    const int strips = (int)e4s_ceil_div(2 * h, wc::BLUR_ROWS);
    const int64_t blocks = e4s_ceil_div((int64_t)batch * strips * w * (cout / 4), wc::BLUR_THREADS);
    E4S_REQUIRE(blocks < (1ll << 31), E4S_ERR_SHAPE);
    wc::convt_blur_kernel<<<(unsigned)blocks, wc::BLUR_THREADS, 0, st>>>(t_buf, fir4x4, demod, noise, noise_w, bias, y, batch, h,
                                                                         w, cout, noise_b, act ? 1 : 0, strips);
    return e4s_launch_status();
}

extern "C" int e4s_modconv3x3_up_masked_tcr_fwd(const float* x, const void* wt_hilo_bf16, const void* w_hilo_bf16,
                                                const float* fir4x4, const float* s, const float* demod, const uint8_t* label,
                                                const float* noise, const float* noise_w, const float* bias, uint32_t* need,
                                                int* base, int* count, uint32_t* rows, float* t_buf, float* y, int batch, int h,
                                                int w, int cin, int cout, int ncls, int cap, int noise_b, int act, void* stream) {
    namespace wc = wgmma_conv;
    E4S_REQUIRE(w_hilo_bf16 && fir4x4 && label && need && base && count && rows && t_buf && cap > 0, E4S_ERR_ARG);
    if (const int rc = wc::check_modconv_fwd(x, wt_hilo_bf16, s, demod, label, noise, noise_w, bias, y, batch, h, w, cin,
                                             cout, ncls, noise_b, h + 1 < (1 << 14) && w + 1 < (1 << wc::ROW_NBITS)))
        return rc;
    E4S_REQUIRE(e4s_aligned16(w_hilo_bf16) && e4s_aligned16(t_buf), E4S_ERR_ALIGN);
    cudaStream_t st = (cudaStream_t)stream;
    wc::convt_row_list_kernel<<<batch, wc::LIST_THREADS, 0, st>>>(label, need, base, count, rows, h, w, ncls, cap);
    if (const int rc = e4s_launch_status()) return rc;
    // GEMM over each sample's rows in blocks of 128; blocks past the list's end cost one load
    wc::Params p{};
    p.a = x, p.wt = static_cast<const __nv_bfloat16*>(wt_hilo_bf16), p.s = s, p.out = t_buf, p.rows = rows, p.row_count = count;
    p.batch = batch, p.h = h, p.w = w, p.kch = cin, p.nch = 4 * cout, p.ncls = ncls, p.cap = cap;
    p.tiles_x = (int)e4s_ceil_div(cap, wc::M);
    const int nt = wc::pick_ntile_rows(cout, (int64_t)p.tiles_x * batch);
    if (const int rc = nt == 128 ? wc::launch_rows<128>(p, st) : nt == 64 ? wc::launch_rows<64>(p, st) : wc::launch_rows<32>(p, st))
        return rc;
    const int64_t blocks = e4s_ceil_div((int64_t)batch * 2 * h * e4s_ceil_div(2 * w, wc::BLUR_PIX) * (cout / 4), wc::BLUR_THREADS);
    E4S_REQUIRE(blocks < (1ll << 31), E4S_ERR_SHAPE);
    wc::convt_blur_masked_kernel<<<(unsigned)blocks, wc::BLUR_THREADS, 0, st>>>(t_buf, need, base, count, label, fir4x4, demod, noise,
                                                                                noise_w, bias, y, batch, h, w, cout, ncls, cap,
                                                                                noise_b, act ? 1 : 0);
    if (const int rc = e4s_launch_status()) return rc;
    // samples whose list overflowed: the folded parity kernel (its items for the other samples return at once)
    wc::Params f{};
    f.a = x, f.wt = static_cast<const __nv_bfloat16*>(w_hilo_bf16), f.s = s, f.demod = demod, f.label = label, f.row_count = count;
    f.noise = noise, f.noise_w = noise_w, f.bias = bias, f.out = y, f.cap = cap;
    f.batch = batch, f.h = h, f.w = w, f.kch = cin, f.nch = cout, f.ncls = ncls, f.noise_b = noise_b, f.act = act ? 1 : 0;
    f.up = 1;
    wc::set_taps(f, 0);
    return wc::forward(f, st);
}

// Arguments common to the two plain-convolution entry points into p; the first failing check gives the error code.
// `extra` is every further pointer of the entry (each may be NULL), checked for 16-byte alignment.
static int plain_conv_params(wgmma_conv::Params& p, const float* x, const void* w_hilo_bf16, const float* scale,
                             const float* shift, float* y, int batch, int h, int w, int cin, int cout, int out_stride,
                             int tap_mask, std::initializer_list<const void*> extra) {
    E4S_REQUIRE(x && w_hilo_bf16 && y, E4S_ERR_ARG);
    E4S_REQUIRE(tap_mask >= 0 && tap_mask <= 0x1FF, E4S_ERR_ARG);
    E4S_REQUIRE(batch > 0 && h > 0 && w > 0 && cin > 0 && cout > 0, E4S_ERR_ARG);
    E4S_REQUIRE((cin % 32) == 0 && (cout % 32) == 0, E4S_ERR_SHAPE);
    E4S_REQUIRE(out_stride == 1 || ((out_stride == 2 || out_stride == 4) && (h % 2) == 0 && (w % 2) == 0), E4S_ERR_SHAPE);
    E4S_REQUIRE(e4s_aligned16(x) && e4s_aligned16(w_hilo_bf16) && e4s_aligned16(y) && (!scale || e4s_aligned16(scale)) &&
                    (!shift || e4s_aligned16(shift)),
                E4S_ERR_ALIGN);
    for (const void* q : extra) E4S_REQUIRE(!q || e4s_aligned16(q), E4S_ERR_ALIGN);
    p.a = x, p.wt = static_cast<const __nv_bfloat16*>(w_hilo_bf16), p.s = scale, p.shift = shift, p.out = y;
    p.batch = batch, p.h = h, p.w = w, p.kch = cin, p.nch = cout, p.ncls = 1;
    p.out_stride = out_stride;
    wgmma_conv::set_taps(p, tap_mask);
    return E4S_OK;
}

extern "C" int e4s_conv3x3_tcr_f32(const float* x, const void* w_hilo_bf16, const float* scale, const float* shift,
                                   const float* prelu_slope, float* y, int batch, int h, int w, int cin, int cout,
                                   int out_stride, int tap_mask, void* stream) {
    wgmma_conv::Params p{};
    if (const int rc = plain_conv_params(p, x, w_hilo_bf16, scale, shift, y, batch, h, w, cin, cout, out_stride, tap_mask,
                                         {prelu_slope}))
        return rc;
    p.slope = prelu_slope, p.act = prelu_slope ? 2 : 0;
    return wgmma_conv::forward(p, (cudaStream_t)stream);
}

extern "C" int e4s_conv3x3_bias_tcr_f32(const float* x, const void* w_hilo_bf16, const float* scale, const float* shift,
                                        const float* bias, const float* residual, float* y, int batch, int h, int w, int cin,
                                        int cout, int out_stride, int tap_mask, int relu, void* stream) {
    wgmma_conv::Params p{};
    if (const int rc = plain_conv_params(p, x, w_hilo_bf16, scale, shift, y, batch, h, w, cin, cout, out_stride, tap_mask,
                                         {bias, residual}))
        return rc;
    p.bias = bias, p.residual = residual, p.act = relu ? 1 : 0;
    return wgmma_conv::forward<wgmma_conv::FWD_BIAS>(p, (cudaStream_t)stream);
}

// The plain-mode entries' checks and parameters (p.reflect = reflect for FWD_REFL); up: the halo reads the input at
// (sy >> up, sx >> up) (nearest up-sampling by 2^up; h, w: the input grid)
static int dense_params(wgmma_conv::Params& p, const float* x, int x_ld, const void* w_hilo_bf16, const float* bias, float alpha,
                        const float* r0, float beta, const float* r1, float* y, int y_ld, int batch, int h, int w, int cin,
                        int cout, int up, int reflect, int tap_mask, float lrelu_slope) {
    E4S_REQUIRE(x && w_hilo_bf16 && y, E4S_ERR_ARG);
    E4S_REQUIRE(batch > 0 && h > 0 && w > 0 && cin > 0 && cout > 0 && x_ld >= cin && y_ld >= cout, E4S_ERR_ARG);
    E4S_REQUIRE(up >= 0 && up <= 2, E4S_ERR_ARG);
    E4S_REQUIRE((cin % 32) == 0 && (cout % 32) == 0, E4S_ERR_SHAPE);
    E4S_REQUIRE((x_ld % 4) == 0 && (y_ld % 4) == 0, E4S_ERR_ALIGN);
    E4S_REQUIRE(e4s_aligned16(x) && e4s_aligned16(w_hilo_bf16) && e4s_aligned16(y), E4S_ERR_ALIGN);
    for (const void* q : {(const void*)bias, (const void*)r0, (const void*)r1}) E4S_REQUIRE(!q || e4s_aligned16(q), E4S_ERR_ALIGN);
    const int m = 1 << up;
    p.a = x, p.wt = static_cast<const __nv_bfloat16*>(w_hilo_bf16), p.bias = bias, p.out = y;
    p.residual = r0, p.residual2 = r1, p.alpha = alpha, p.beta = beta, p.lrelu = lrelu_slope;
    p.a_ld = x_ld, p.out_ld = y_ld, p.up = up, p.reflect = reflect;
    p.batch = batch, p.h = h * m, p.w = w * m, p.kch = cin, p.nch = cout, p.ncls = 1;
    wgmma_conv::set_taps(p, tap_mask);
    wgmma_conv::tiles(p);
    return E4S_OK;
}

// The plain-mode entries: checks, then the launch of MODE (FWD_DENSE: zero padding; FWD_REFL: p.reflect = reflect) at N
// tile ntile (0: pick_ntile's choice for the launch size).
template <int MODE>
static int dense_conv(const float* x, int x_ld, const void* w_hilo_bf16, const float* bias, float alpha, const float* r0,
                      float beta, const float* r1, float* y, int y_ld, int batch, int h, int w, int cin, int cout, int up,
                      int reflect, int tap_mask, float lrelu_slope, void* stream, int ntile = 0) {
    wgmma_conv::Params p{};
    if (const int rc = dense_params(p, x, x_ld, w_hilo_bf16, bias, alpha, r0, beta, r1, y, y_ld, batch, h, w, cin, cout, up,
                                    reflect, tap_mask, lrelu_slope))
        return rc;
    const int nt = ntile ? ntile : wgmma_conv::pick_ntile(cout, (int64_t)p.tiles_x * p.tiles_y * batch);
    return wgmma_conv::launch<MODE>(p, nt, 1, (cudaStream_t)stream);
}

extern "C" int e4s_conv3x3_dense_tcr_f32(const float* x, int x_ld, const void* w_hilo_bf16, const float* bias, float alpha,
                                         const float* r0, float beta, const float* r1, float* y, int y_ld, int batch, int h,
                                         int w, int cin, int cout, int up, float lrelu_slope, void* stream) {
    return dense_conv<wgmma_conv::FWD_DENSE>(x, x_ld, w_hilo_bf16, bias, alpha, r0, beta, r1, y, y_ld, batch, h, w, cin, cout,
                                             up ? 1 : 0, 0, 0, lrelu_slope, stream);
}

extern "C" int e4s_conv3x3_reflect_tcr_f32(const float* x, int x_ld, const void* w_hilo_bf16, const float* bias, float alpha,
                                           const float* r0, float beta, const float* r1, float* y, int y_ld, int batch, int h,
                                           int w, int cin, int cout, int mode, float lrelu_slope, void* stream) {
    E4S_REQUIRE(mode >= 0 && mode <= 2, E4S_ERR_ARG);
    E4S_REQUIRE(h >= 2 && w >= 2, E4S_ERR_SHAPE);
    // mode 0: stride 1, mirror; 1: nearest 2x up-sampling, replicate; 2: stride 2 over the space-to-depth operand (taps
    // {-1, 0}^2), replicate
    return dense_conv<wgmma_conv::FWD_REFL>(x, x_ld, w_hilo_bf16, bias, alpha, r0, beta, r1, y, y_ld, batch, h, w, cin, cout,
                                            mode == 1, mode == 0 ? 1 : 2, mode == 2 ? 0x1B : 0, lrelu_slope, stream);
}

extern "C" int e4s_conv3x3_zero_tcr_f32(const float* x, int x_ld, const void* w_hilo_bf16, const float* bias, float alpha,
                                        const float* r0, float beta, const float* r1, float* y, int y_ld, int batch, int h, int w,
                                        int cin, int cout, int stride, float lrelu_slope, void* stream) {
    E4S_REQUIRE(stride == 1 || stride == 2, E4S_ERR_ARG);
    // zero padding 1; stride 2 over the space-to-depth operand: the taps (dy, dx) in {-1, 0}^2.  The N tile follows the
    // channel count only, so each output's sum order (and value) does not depend on the batch
    return dense_conv<wgmma_conv::FWD_DENSE>(x, x_ld, w_hilo_bf16, bias, alpha, r0, beta, r1, y, y_ld, batch, h, w, cin, cout,
                                             0, 0, stride == 2 ? 0x1B : 0, lrelu_slope, stream, (cout % 64) == 0 ? 64 : 32);
}

extern "C" int e4s_conv3x3_zero_up_tcr_f32(const float* x, int x_ld, const void* w_hilo_bf16, const float* bias, float* y,
                                           int y_ld, int batch, int h, int w, int cin, int cout, int up_shift, float lrelu_slope,
                                           void* stream) {
    E4S_REQUIRE(up_shift == 1 || up_shift == 2, E4S_ERR_ARG);
    // e4s_conv3x3_zero_tcr_f32 over the nearest up-sampling of x by 2^up_shift, read through the halo copy (the
    // up-sampled input is never written); the N tile follows the channel count only
    return dense_conv<wgmma_conv::FWD_DENSE>(x, x_ld, w_hilo_bf16, bias, 1.f, nullptr, 1.f, nullptr, y, y_ld, batch, h, w, cin,
                                             cout, up_shift, 0, 0, lrelu_slope, stream, (cout % 64) == 0 ? 64 : 32);
}

extern "C" int e4s_spade_tcr_f32(const float* actv, int actv_ld, const void* w_hilo_bf16, const float* bias, const float* x,
                                 int x_ld, int x_half, const float* scale, const float* shift, float* y, int y_ld, int batch,
                                 int h, int w, int cin, int c, float lrelu_slope, void* stream) {
    E4S_REQUIRE(bias && x && scale && shift && x_ld >= c && y_ld >= c && (x_half == 0 || x_half == 1), E4S_ERR_ARG);
    E4S_REQUIRE(!x_half || ((h % 2) == 0 && (w % 2) == 0), E4S_ERR_SHAPE);
    wgmma_conv::Params p{};
    // the GEMM's 2 C columns are the (gamma, beta) pairs; its output pitch is unused (the epilogue stores C channels)
    if (const int rc = dense_params(p, actv, actv_ld, w_hilo_bf16, bias, 1.f, nullptr, 1.f, nullptr, y, 2 * c, batch, h, w, cin,
                                    2 * c, 0, 0, 0, lrelu_slope))
        return rc;
    p.out_ld = y_ld, p.norm_x = x, p.norm_ld = x_ld, p.norm_half = x_half, p.s = scale, p.shift = shift;
    // the N tile follows the channel count only: bit identical at any batch
    return wgmma_conv::launch<wgmma_conv::FWD_SPADE>(p, (2 * c) % 64 == 0 ? 64 : 32, 1, (cudaStream_t)stream);
}

// The pointwise entries' checks and parameters
static int pw_params(wgmma_conv::Params& p, const float* x, int x_ld, const void* w_hilo_bf16, const float* bias, float alpha,
                     const float* r0, const float* r_up, int r_up_ld, float* y, int y_ld, int batch, int h, int w, int cin,
                     int cout, int stride, float lrelu_slope) {
    E4S_REQUIRE(x && w_hilo_bf16 && y, E4S_ERR_ARG);
    E4S_REQUIRE(batch > 0 && h > 0 && w > 0 && cin > 0 && cout > 0 && x_ld >= cin && y_ld >= cout, E4S_ERR_ARG);
    E4S_REQUIRE(stride == 1 || stride == 2, E4S_ERR_ARG);
    E4S_REQUIRE(!r_up || r_up_ld >= cout, E4S_ERR_ARG);
    E4S_REQUIRE((cin % 32) == 0 && (cout % 32) == 0 && (!r_up || ((h % 2) == 0 && (w % 2) == 0)), E4S_ERR_SHAPE);
    E4S_REQUIRE((x_ld % 4) == 0 && (y_ld % 4) == 0 && (!r_up || (r_up_ld % 4) == 0), E4S_ERR_ALIGN);
    E4S_REQUIRE(e4s_aligned16(x) && e4s_aligned16(w_hilo_bf16) && e4s_aligned16(y), E4S_ERR_ALIGN);
    for (const void* q : {(const void*)bias, (const void*)r0, (const void*)r_up}) E4S_REQUIRE(!q || e4s_aligned16(q), E4S_ERR_ALIGN);
    p.a = x, p.wt = static_cast<const __nv_bfloat16*>(w_hilo_bf16), p.bias = bias, p.out = y;
    p.residual = r0, p.residual_up = r_up, p.rup_ld = r_up_ld, p.alpha = alpha, p.beta = 1.f, p.lrelu = lrelu_slope;
    p.a_ld = x_ld, p.out_ld = y_ld, p.in_stride = stride;
    p.batch = batch, p.h = h * stride, p.w = w * stride, p.mh = h, p.mw = w, p.kch = cin, p.nch = cout, p.ncls = 1;
    // K chunks per ring slot: four (eight K16 slices per barrier) where Cin allows it
    p.ntaps = (cin % 128) == 0 ? 4 : (cin % 64) == 0 ? 2 : 1;
    for (int i = 0; i < p.ntaps; ++i) p.taps[i] = i;
    wgmma_conv::tiles(p);
    return E4S_OK;
}

extern "C" int e4s_conv1x1_tcr_f32(const float* x, int x_ld, const void* w_hilo_bf16, const float* bias, float alpha,
                                   const float* r0, const float* r_up, int r_up_ld, float* y, int y_ld, int batch, int h, int w,
                                   int cin, int cout, int stride, float lrelu_slope, void* stream) {
    wgmma_conv::Params p{};
    if (const int rc = pw_params(p, x, x_ld, w_hilo_bf16, bias, alpha, r0, r_up, r_up_ld, y, y_ld, batch, h, w, cin, cout, stride,
                                 lrelu_slope))
        return rc;
    // the N tile (and with it each output's sum order) follows the channel count only: bit identical at any batch
    return wgmma_conv::launch<wgmma_conv::FWD_PW>(p, (cout % 64) == 0 ? 64 : 32, 1, (cudaStream_t)stream);
}

extern "C" int e4s_conv1x1_factor_tcr_f32(const float* x, int x_ld, const void* w_hilo_bf16, const float* bias,
                                          const float* factor, float* y, int y_ld, int batch, int h, int w, int cin, int cout,
                                          void* stream) {
    E4S_REQUIRE(factor, E4S_ERR_ARG);
    wgmma_conv::Params p{};
    if (const int rc = pw_params(p, x, x_ld, w_hilo_bf16, bias, 1.f, nullptr, nullptr, 0, y, y_ld, batch, h, w, cin, cout, 1, 1.f))
        return rc;
    p.factor = factor;
    return wgmma_conv::launch<wgmma_conv::FWD_PWF>(p, (cout % 64) == 0 ? 64 : 32, 1, (cudaStream_t)stream);
}

// The mosaic of a volumetric launch (VolGrid): gutterless stacked slices when the tiles fit them exactly, else cells with
// one-pixel zero gutters, 16 to a mosaic row (16 (W + 1) columns: a whole number of 16-pixel tiles).  Returns the mosaic
// size (rows, columns) in mh, mw.
static wgmma_conv::VolGrid vol_grid(int batch, int depth, int ho, int wo, int& mh, int& mw) {
    using namespace wgmma_conv;
    VolGrid v{};
    v.depth = depth, v.cells = batch * depth;
    v.gutter = (ho % TH) == 0 && (wo % TW) == 0 ? 0 : 1;
    v.ncx = v.gutter ? 16 : 1;
    mh = (int)e4s_ceil_div(v.cells, v.ncx) * (ho + v.gutter), mw = v.ncx * (wo + v.gutter);
    return v;
}

extern "C" int e4s_conv3d_tcr_plan(int batch, int depth, int ho, int wo, int* mosaic_h, int* mosaic_w) {
    E4S_REQUIRE(batch > 0 && depth > 0 && ho > 0 && wo > 0 && mosaic_h && mosaic_w, E4S_ERR_ARG);
    vol_grid(batch, depth, ho, wo, *mosaic_h, *mosaic_w);
    return E4S_OK;
}

// The volumetric entries: x, y channel slices of [B, *, *, D, *] buffers with voxel pitches x_vp, y_vp (floats)
// (r0: added after the bias, before the ReLU, pitched like y, or NULL)
static int conv3d(const float* x, int x_vp, const void* w_hilo_bf16, const float* bias, float* y, int y_vp, int batch, int depth,
                  int h, int w, int cin, int cout, int up, int relu, void* stream, const float* r0 = nullptr) {
    E4S_REQUIRE(x && w_hilo_bf16 && y, E4S_ERR_ARG);
    E4S_REQUIRE(batch > 0 && depth > 0 && h > 0 && w > 0 && cin > 0 && cout > 0 && x_vp >= cin && y_vp >= cout, E4S_ERR_ARG);
    E4S_REQUIRE((cin % 32) == 0 && (cout % 32) == 0, E4S_ERR_SHAPE);
    E4S_REQUIRE((x_vp % 4) == 0 && (y_vp % 4) == 0, E4S_ERR_ALIGN);
    E4S_REQUIRE(e4s_aligned16(x) && e4s_aligned16(w_hilo_bf16) && e4s_aligned16(y) && (!bias || e4s_aligned16(bias)) &&
                    (!r0 || e4s_aligned16(r0)),
                E4S_ERR_ALIGN);
    const int m = up ? 2 : 1;
    // 32-bit index arithmetic inside a sample and the mosaic
    E4S_REQUIRE((int64_t)h * m * w * m * depth * (x_vp > y_vp ? x_vp : y_vp) < (1ll << 31) &&
                    (int64_t)batch * depth * (h * m + 1) * (w * m + 1) < (1ll << 30),
                E4S_ERR_SHAPE);
    wgmma_conv::Params p{};
    p.a = x, p.wt = static_cast<const __nv_bfloat16*>(w_hilo_bf16), p.bias = bias, p.out = y;
    p.alpha = 1.f, p.beta = 1.f, p.lrelu = relu ? 0.f : 1.f, p.residual = r0;
    p.a_ld = depth * x_vp, p.out_ld = depth * y_vp, p.vox_in = x_vp, p.vox_out = y_vp, p.up = up ? 1 : 0;
    p.batch = 1, p.h = h * m, p.w = w * m, p.kch = 3 * cin, p.nch = cout, p.ncls = 1;
    p.vol = vol_grid(batch, depth, h * m, w * m, p.mh, p.mw);
    wgmma_conv::set_taps(p, 0);
    wgmma_conv::tiles(p);
    // the N tile (and with it each output's sum order) follows the channel count only: bit identical at any batch
    return wgmma_conv::launch<wgmma_conv::FWD_VOL>(p, (cout % 64) == 0 ? 64 : 32, 1, (cudaStream_t)stream);
}

extern "C" int e4s_conv3d_tcr_f32(const float* x, const void* w_hilo_bf16, const float* bias, float* y, int batch, int depth,
                                  int h, int w, int cin, int cout, int up, int relu, void* stream) {
    return conv3d(x, cin, w_hilo_bf16, bias, y, cout, batch, depth, h, w, cin, cout, up, relu, stream);
}

extern "C" int e4s_conv3d_pitched_tcr_f32(const float* x, int x_vp, const void* w_hilo_bf16, const float* bias, float* y, int y_vp,
                                          int batch, int depth, int h, int w, int cin, int cout, int up, int relu, void* stream) {
    return conv3d(x, x_vp, w_hilo_bf16, bias, y, y_vp, batch, depth, h, w, cin, cout, up, relu, stream);
}

extern "C" int e4s_conv3d_residual_tcr_f32(const float* x, const void* w_hilo_bf16, const float* bias, const float* residual,
                                           float* y, int batch, int depth, int h, int w, int cin, int cout, int relu, void* stream) {
    E4S_REQUIRE(residual, E4S_ERR_ARG);
    return conv3d(x, cin, w_hilo_bf16, bias, y, cout, batch, depth, h, w, cin, cout, 0, relu, stream, residual);
}

extern "C" int e4s_conv7x7_slices_tcr_f32(const float* x, const void* w_hilo_bf16, float* y, int batch, int depth, int h, int w,
                                          int cin, void* stream) {
    using namespace wgmma_conv;
    E4S_REQUIRE(x && w_hilo_bf16 && y, E4S_ERR_ARG);
    E4S_REQUIRE(batch > 0 && depth > 0 && h > 0 && w > 0 && cin > 0, E4S_ERR_ARG);
    E4S_REQUIRE((cin % KC) == 0 && (h % TH) == 0 && (w % TW) == 0 && batch <= 65535 && depth <= 65535, E4S_ERR_SHAPE);
    E4S_REQUIRE(e4s_aligned16(x) && e4s_aligned16(w_hilo_bf16) && e4s_aligned16(y), E4S_ERR_ALIGN);
    const int tiles_x = w / TW;
    static E4sSmemOptIn optin;
    if (const int rc = e4s_smem_optin(optin, conv7x7_slices_kernel, K7_SMEM)) return rc;
    conv7x7_slices_kernel<<<dim3((unsigned)(tiles_x * (h / TH)), (unsigned)depth, (unsigned)batch), NUM_THREADS, K7_SMEM,
                            (cudaStream_t)stream>>>(x, static_cast<const __nv_bfloat16*>(w_hilo_bf16), y, depth, h, w, cin,
                                                    tiles_x);
    return e4s_launch_status();
}

extern "C" int e4s_modconv3x3_bwd_tc(const float* gy, const float* y, const float* x, const void* wd_hilo_bf16, const float* s,
                                     const float* demod, const uint8_t* label, float* gx, float* gs, int batch, int h, int w,
                                     int cin, int cout, int ncls, int up, int act, void* stream) {
    E4S_REQUIRE(gy && wd_hilo_bf16 && s && (gx || gs), E4S_ERR_ARG);
    E4S_REQUIRE(!act || y, E4S_ERR_ARG);
    E4S_REQUIRE(!gs || x, E4S_ERR_ARG);
    E4S_REQUIRE(batch > 0 && h > 0 && w > 0 && cin > 0 && cout > 0 && ncls > 0 && ncls <= 32, E4S_ERR_ARG);
    E4S_REQUIRE((cin % 32) == 0 && (cout % 32) == 0, E4S_ERR_SHAPE);
    E4S_REQUIRE(label || ncls == 1, E4S_ERR_ARG);
    cudaStream_t st = (cudaStream_t)stream;
    wgmma_conv::Params p{};
    p.a = gy, p.y = act ? y : nullptr, p.x = x, p.wt = static_cast<const __nv_bfloat16*>(wd_hilo_bf16), p.s = s, p.demod = demod;
    p.label = label, p.out = gx, p.gs = gs;
    p.batch = batch, p.h = h, p.w = w, p.kch = cout, p.nch = cin, p.ncls = ncls, p.act = act ? 1 : 0;
    p.up = up ? 1 : 0;
    wgmma_conv::set_taps(p, 0);
    wgmma_conv::tiles(p);
    const int nph = up ? 4 : 1;
    const int64_t pixel_tiles = (int64_t)p.tiles_x * p.tiles_y * batch;
    const int nt = wgmma_conv::pick_ntile(cin, pixel_tiles);
    wgmma_conv::choose_split(pixel_tiles * (cin / nt), label ? ncls : 1, nph, p.gsplit, p.hsplit);
    p.atomic_gx = p.gsplit * p.hsplit > 1;
    if (p.atomic_gx && gx && cudaMemsetAsync(gx, 0, (size_t)batch * h * w * cin * sizeof(float), st) != cudaSuccess)
        return (int)cudaGetLastError();
    return wgmma_conv::launch<wgmma_conv::BWD>(p, nt, (int64_t)p.gsplit * p.hsplit, st);
}

// Host-only: the work list e4s_modconv3x3_bwd_tc builds for this shape (N-tile width, region-pass and parity-plane split).
// ncls = number of regions the label map can hold (1 without one).  No launch, no device access beyond the SM count
// (132 when no device is present) - lets the host-side heuristics be tested without a GPU.
extern "C" int e4s_modconv3x3_bwd_tc_plan(int batch, int h, int w, int cin, int ncls, int up, int* ntile, int* gsplit, int* hsplit) {
    E4S_REQUIRE(ntile && gsplit && hsplit && batch > 0 && h > 0 && w > 0 && cin > 0 && ncls > 0 && ncls <= 32, E4S_ERR_ARG);
    E4S_REQUIRE((cin % 32) == 0, E4S_ERR_SHAPE);
    const int64_t pixel_tiles = e4s_ceil_div(w, wgmma_conv::TW) * e4s_ceil_div(h, wgmma_conv::TH) * batch;
    *ntile = wgmma_conv::pick_ntile(cin, pixel_tiles);
    wgmma_conv::choose_split(pixel_tiles * (cin / *ntile), ncls, up ? 4 : 1, *gsplit, *hsplit);
    return E4S_OK;
}
