// Tensor-core 3x3 convolutions of the library (sm_90a): what more than one of their kernel families uses.
//   wgmma_conv_smem.cu  conv3x3_wgmma_kernel, both operands staged in shared memory: the folded up-sampling forward, the
//                       encoder's convolution, the BiSeNet bias convolution and the modulated convolution's gradient;
//   wgmma_conv_rs.cu    conv3x3_rs_kernel, the A operand built in registers from fp32 halo tiles: the plain modulated
//                       layers and the plain, reflect-padded, 1x1, SPADE and volumetric convolutions; conv7x7_slices_kernel;
//   wgmma_convt.cu      the up-sampling layers' transposed-convolution GEMMs on register operands (convt_rs_kernel
//                       unmasked, rows_rs_kernel over (pixel, region) rows when masked), their blur passes and row list.
// The kernels share the split-precision MMA step (split_mma, SplitAcc), the work-item decode (decode_item) and the layer
// epilogue (epilogue2); the register-operand kernels share the swizzled fp32 tile (tile_at), the fragment build
// (build_frag) and the K step (issue_rs).
#pragma once
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

// The MODE template argument of a kernel.  conv3x3_wgmma_kernel:
// FWD: the folded forward and the encoder's convolution, epilogue2.
// FWD_BIAS: FWD with the epilogue relu?(acc + bias + residual) (epilogue_bias2) in place of epilogue2.
// BWD: the input / style gradient of the modulated convolution.
// conv3x3_rs_kernel:
// FWD_RS: the plain modulated convolution (styles of each row's region), epilogue2.
// FWD_DENSE: the plain convolution: unscaled pitched operands, the ESRGAN epilogue.
// FWD_REFL: FWD_DENSE with reflection padding in the halo copy (Params::reflect) in place of the zero fill.
// FWD_PW: FWD_DENSE as a 1x1 (pointwise) convolution: no halo, several K chunks per ring slot (Params::in_stride, r_up).
// FWD_VOL: FWD_DENSE as a 3x3x3 convolution over a mosaic of depth slices (VolGrid).
// FWD_SPADE: FWD_DENSE whose output columns are interleaved (gamma, beta) pairs of a SPADE modulation, applied in the
// epilogue to the instance-normalised input (Params::norm_x); neither the normalised input nor gamma / beta is written.
// FWD_PWF: FWD_PW with the result multiplied by a per-pixel factor (Params::factor).
enum Mode { FWD = 0, BWD = 2, FWD_RS = 3, FWD_BIAS = 4, FWD_DENSE = 5, FWD_REFL = 6, FWD_PW = 7, FWD_VOL = 8,
            FWD_SPADE = 9, FWD_PWF = 10 };

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
    // rows_rs_kernel: row i of sample b is the packed (m, n, region) rows[b * cap + i], out is [B, cap, nch];
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
__device__ __forceinline__ float4 ld4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }

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

// The register-operand kernels' fp32 A tiles in shared memory (a halo tile, pixel tiles or gathered rows): pixel hp at
// hp * 128 bytes, its 16-byte channel quad c at (c ^ (hp % 8)) * 16.  The 8 fragment rows of a warp are 8 consecutive
// pixels, so the XOR spreads their reads over all 32 banks (each 256-byte float2 read of a warp is served in the minimal
// two wavefronts).
// tile_at(tile, hp, c): the address of that quad in the tile at `tile` (a shared-memory address or a pointer)
template <typename T>
__device__ __forceinline__ T tile_at(T tile, int hp, int c) { return tile + hp * 128 + ((c ^ (hp & 7)) << 4); }

// x_hi / x_lo fragments of K16 slice ks from such a tile, for the thread with lane % 4 = q: register r is fragment row
// h = r & 1 at the tile's pixel hp(h), channels 16 ks + 8 (r >> 1) + 2 q, + 1, multiplied by that row's styles (s0 for
// row 0, s1 for row 1, element 2 ks + (r >> 1)) unless they are null
template <typename Pixel>
__device__ __forceinline__ void build_frag(const uint8_t* tile, Pixel hp, int q, int ks, uint32_t (&hi)[4], uint32_t (&lo)[4],
                                           const float2* s0 = nullptr, const float2* s1 = nullptr) {
#pragma unroll
    for (int r = 0; r < 4; ++r) {
        const int h = r & 1, j = 2 * ks + (r >> 1);
        const float2 v = *reinterpret_cast<const float2*>(tile_at(tile, hp(h), 2 * j + (q >> 1)) + (q & 1) * 8);
        if (s0) {
            const float2 sv = h ? s1[j] : s0[j];
            split2(v.x * sv.x, v.y * sv.y, hi[r], lo[r]);
        } else {
            split2(v.x, v.y, hi[r], lo[r]);
        }
    }
}

// One K step of a register-operand kernel: both K16 slices' split products of fragments hi / lo and the B tiles at bt
// (w_hi, w_lo NT * KC * 2 bytes on; slice ks at + ks * 2 LBO); first: the step starts the accumulation
template <int NT>
__device__ __forceinline__ void issue_rs(SplitAcc<NT>& acc, uint32_t (&hi)[2][4], uint32_t (&lo)[2][4], uint32_t bt, bool first) {
    acc.fence();
    fence_frag(hi);
    fence_frag(lo);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 2; ++ks) {
        const uint32_t bh = bt + ks * 2 * LBO;
        split_mma(acc, hi[ks], lo[ks], bh, bh + NT * KC * 2, (first && ks == 0) ? 0 : 1);
    }
    wgmma_commit();
    acc.fence();
    fence_frag(hi);
    fence_frag(lo);
}

// ------------------------------------------------------------------------------------------ host
inline int num_sms() { return e4s_num_sms(); }

// N-tile width (output channels per work item): 64 when the channel count allows it and the launch still has work for
// half the SMs, else 32.  E4S_B200_NTILE=32|64 forces a width the channel count allows.
inline int pick_ntile(int channels, int64_t items_per_ntile_column) {
    if (const char* f = getenv("E4S_B200_NTILE")) {
        const int v = atoi(f);
        if ((v == 32 || v == 64) && channels % v == 0) return v;
    }
    if (channels % 64 != 0) return 32;
    return items_per_ntile_column * (channels / 64) >= num_sms() / 2 ? 64 : 32;
}

inline void set_taps(Params& p, int tap_mask) {
    p.ntaps = 0;
    for (int t = 0; t < 9; ++t)
        if (!tap_mask || ((tap_mask >> t) & 1)) p.taps[p.ntaps++] = t;
}

// pixel tiles over the output row grid (the input grid unless the caller set another one)
inline void tiles(Params& p) {
    if (!p.mh) p.mh = p.h, p.mw = p.w;
    p.tiles_x = (int)e4s_ceil_div(p.mw, TW);
    p.tiles_y = (int)e4s_ceil_div(p.mh, TH);
}

// Argument checks of the modulated forward entries; the first failing one gives the error code.  ok_shape: the entry's
// own shape limits.
inline int check_modconv_fwd(const float* x, const void* w_hilo, const float* s, const float* demod, const uint8_t* label,
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

// The folded forward on conv3x3_wgmma_kernel (MODE FWD or FWD_BIAS; wgmma_conv_smem.cu)
template <int MODE = FWD>
int forward(Params p, cudaStream_t st);

}  // namespace wgmma_conv
