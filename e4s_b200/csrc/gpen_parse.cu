// The RGB-side convolutions of GPEN's ParseNet (src/pretrained/gpen/face_parse/parse_model.py): encoder.0 (3 -> 64,
// planar image in, pixel-major features out), out_img_conv (64 -> 3, planar image out) and out_mask_conv (64 -> 19) fused
// with the first-index argmax over the classes and the MASK_COLORMAP lookup.  All 3x3, stride 1, reflection padding 1,
// + bias; they are 1.6 % of the network's multiply-adds, every other convolution runs on the tensor-core kernel
// (e4s_conv3x3_reflect_tcr_f32).  fp32 on CUDA cores: a thread computes every output channel of one pixel, the weights
// from shared memory (a broadcast: every thread of a warp reads the same word).  Each output sums taps row-major, channels
// ascending, then adds the bias (bit reproducible).
//
// encoder.0 can also take FaceParse.process_tensor's raw input (BGR in [0, 1], any size): the channel flip, v * 2 - 1 and
// F.interpolate(mode='nearest') to the network's size happen as the pixels are read, with the same fp32 arithmetic.
#include "common.cuh"

namespace gparse {

constexpr int THREADS = 128;          // pixels of one image row per CTA

// reflection padding 1: row -1 reads row 1, row n reads row n - 2
__device__ __forceinline__ int reflect1(int i, int n) { return i < 0 ? -i : (i >= n ? 2 * n - 2 - i : i); }

// F.interpolate(mode='nearest') source index of output index d: min(floor(d * scale), n_in - 1), scale = n_in / n_out in fp32
__device__ __forceinline__ int nearest_src(int d, float scale, int n_in) { return min((int)floorf((float)d * scale), n_in - 1); }

// x planar [B, 3, hs, ws] -> y pixel-major [B, h, w, 64] (pitch y_ld).  PREP: x is BGR in [0, 1] at hs x ws and the
// network input is flip(x) * 2 - 1 resized (nearest) to h x w; else hs == h, ws == w and x is the network input.
template <bool PREP>
__global__ void __launch_bounds__(THREADS) conv_in_kernel(const float* __restrict__ x, int hs, int ws, float scy, float scx,
                                                          const float* __restrict__ wt, const float* __restrict__ bias,
                                                          float* __restrict__ y, int y_ld, int h, int w) {
    constexpr int CIN = 3, COUT = 64;
    __shared__ __align__(16) float sw[9 * CIN * COUT];       // [tap][ci][co]
    __shared__ float sb[COUT];
    for (int e = threadIdx.x; e < 9 * CIN * COUT; e += THREADS) {
        const int tap = e / (COUT * CIN), co = e % COUT, ci = (e / COUT) % CIN;
        sw[e] = __ldg(wt + (co * CIN + ci) * 9 + tap);
    }
    if (threadIdx.x < COUT) sb[threadIdx.x] = __ldg(bias + threadIdx.x);
    __syncthreads();
    const int ox = blockIdx.x * THREADS + threadIdx.x, oy = blockIdx.y, b = blockIdx.z;
    if (ox >= w) return;
    float acc[COUT];
#pragma unroll
    for (int co = 0; co < COUT; ++co) acc[co] = 0.f;
#pragma unroll
    for (int tap = 0; tap < 9; ++tap) {
        int sy = reflect1(oy + tap / 3 - 1, h), sx = reflect1(ox + tap % 3 - 1, w);
        if (PREP) sy = nearest_src(sy, scy, hs), sx = nearest_src(sx, scx, ws);
#pragma unroll
        for (int ci = 0; ci < CIN; ++ci) {
            float v = __ldg(x + (((int64_t)b * CIN + (PREP ? CIN - 1 - ci : ci)) * hs + sy) * ws + sx);
            if (PREP) v = v * 2.f - 1.f;
            const float* wr = sw + (tap * CIN + ci) * COUT;
#pragma unroll
            for (int co = 0; co < COUT; ++co) acc[co] = fmaf(v, wr[co], acc[co]);
        }
    }
    float* yp = y + (((int64_t)b * h + oy) * w + ox) * y_ld;
#pragma unroll
    for (int c4 = 0; c4 < COUT / 4; ++c4)
        reinterpret_cast<float4*>(yp)[c4] = make_float4(acc[4 * c4] + sb[4 * c4], acc[4 * c4 + 1] + sb[4 * c4 + 1],
                                                        acc[4 * c4 + 2] + sb[4 * c4 + 2], acc[4 * c4 + 3] + sb[4 * c4 + 3]);
}

// x pixel-major [B, h, w, 64] (pitch x_ld) -> COUT outputs per pixel.  COUT 3 (out_img_conv): y planar [B, 3, h, w].
// COUT 19 (out_mask_conv): logits planar [B, 19, h, w] when given; the first-index argmax k of the 19 values (a tie keeps
// the lower class) gives lut[k] to mask_u8 [B, h, w] and / or mask_i64 [B, h, w] when given.
template <int COUT>
__global__ void __launch_bounds__(THREADS) conv_out_kernel(const float* __restrict__ x, int x_ld, const float* __restrict__ wt,
                                                           const float* __restrict__ bias, const uint8_t* __restrict__ lut,
                                                           float* __restrict__ y, uint8_t* __restrict__ mask_u8,
                                                           int64_t* __restrict__ mask_i64, int h, int w) {
    constexpr int CIN = 64;
    __shared__ __align__(16) float sw[9 * COUT * CIN];       // [tap][co][ci]: float4 weight reads along the channels
    __shared__ float sb[COUT];
    for (int e = threadIdx.x; e < 9 * CIN * COUT; e += THREADS) {
        const int tap = e / (COUT * CIN), co = (e / CIN) % COUT, ci = e % CIN;
        sw[e] = __ldg(wt + (co * CIN + ci) * 9 + tap);
    }
    if (threadIdx.x < COUT) sb[threadIdx.x] = __ldg(bias + threadIdx.x);
    __syncthreads();
    const int ox = blockIdx.x * THREADS + threadIdx.x, oy = blockIdx.y, b = blockIdx.z;
    if (ox >= w) return;
    float acc[COUT];
#pragma unroll
    for (int co = 0; co < COUT; ++co) acc[co] = 0.f;
#pragma unroll 1
    for (int tap = 0; tap < 9; ++tap) {
        const int sy = reflect1(oy + tap / 3 - 1, h), sx = reflect1(ox + tap % 3 - 1, w);
        const float4* xp = reinterpret_cast<const float4*>(x + (((int64_t)b * h + sy) * w + sx) * x_ld);
#pragma unroll 4
        for (int c4 = 0; c4 < CIN / 4; ++c4) {
            const float4 v = __ldg(xp + c4);
#pragma unroll
            for (int co = 0; co < COUT; ++co) {
                const float4 wv = *reinterpret_cast<const float4*>(sw + (tap * COUT + co) * CIN + 4 * c4);
                acc[co] = fmaf(v.w, wv.w, fmaf(v.z, wv.z, fmaf(v.y, wv.y, fmaf(v.x, wv.x, acc[co]))));
            }
        }
    }
    const int64_t plane = (int64_t)h * w, pix = (int64_t)oy * w + ox;
    float best = 0.f;
    int arg = 0;
#pragma unroll
    for (int co = 0; co < COUT; ++co) {
        const float v = acc[co] + sb[co];
        if (y) y[((int64_t)b * COUT + co) * plane + pix] = v;
        if (co == 0 || v > best) best = v, arg = co;
    }
    if (COUT > 3) {
        const uint8_t m = __ldg(lut + arg);
        if (mask_u8) mask_u8[(int64_t)b * plane + pix] = m;
        if (mask_i64) mask_i64[(int64_t)b * plane + pix] = m;
    }
}

}  // namespace gparse

extern "C" int e4s_conv3x3_rgb_reflect_f32(const float* x, int x_ld, int hs, int ws, int prep, const float* w3x3,
                                           const float* bias, float* y, int y_ld, int batch, int h, int w, int cin, int cout,
                                           void* stream) {
    E4S_REQUIRE(x && w3x3 && bias && y && batch > 0 && h > 1 && w > 1, E4S_ERR_ARG);
    E4S_REQUIRE(((cin == 3 && cout == 64) || (cin == 64 && cout == 3)) && batch < 65536 && h < 65536, E4S_ERR_SHAPE);
    if (cin == 3) {
        E4S_REQUIRE(y_ld >= cout && (prep ? hs > 0 && ws > 0 : hs == h && ws == w), E4S_ERR_ARG);
        E4S_REQUIRE(y_ld % 4 == 0 && e4s_aligned16(y), E4S_ERR_ALIGN);
    } else {
        E4S_REQUIRE(x_ld >= cin && !prep, E4S_ERR_ARG);
        E4S_REQUIRE(x_ld % 4 == 0 && e4s_aligned16(x), E4S_ERR_ALIGN);
    }
    const dim3 grid((unsigned)e4s_ceil_div(w, gparse::THREADS), (unsigned)h, (unsigned)batch);
    cudaStream_t st = (cudaStream_t)stream;
    if (cin == 3 && prep)
        gparse::conv_in_kernel<true><<<grid, gparse::THREADS, 0, st>>>(x, hs, ws, (float)hs / (float)h, (float)ws / (float)w,
                                                                        w3x3, bias, y, y_ld, h, w);
    else if (cin == 3)
        gparse::conv_in_kernel<false><<<grid, gparse::THREADS, 0, st>>>(x, h, w, 1.f, 1.f, w3x3, bias, y, y_ld, h, w);
    else
        gparse::conv_out_kernel<3><<<grid, gparse::THREADS, 0, st>>>(x, x_ld, w3x3, bias, nullptr, y, nullptr, nullptr, h, w);
    return e4s_launch_status();
}

extern "C" int e4s_gpen_parse_head_u8(const float* x, int x_ld, const float* w3x3, const float* bias, const uint8_t* lut,
                                      float* logits, uint8_t* mask_u8, int64_t* mask_i64, int batch, int h, int w, int cin,
                                      int ncls, void* stream) {
    E4S_REQUIRE(x && w3x3 && bias && lut && (logits || mask_u8 || mask_i64) && batch > 0 && h > 1 && w > 1, E4S_ERR_ARG);
    E4S_REQUIRE(cin == 64 && ncls == 19 && batch < 65536 && h < 65536, E4S_ERR_SHAPE);
    E4S_REQUIRE(x_ld >= cin, E4S_ERR_ARG);
    E4S_REQUIRE(x_ld % 4 == 0 && e4s_aligned16(x), E4S_ERR_ALIGN);
    const dim3 grid((unsigned)e4s_ceil_div(w, gparse::THREADS), (unsigned)h, (unsigned)batch);
    gparse::conv_out_kernel<19><<<grid, gparse::THREADS, 0, (cudaStream_t)stream>>>(x, x_ld, w3x3, bias, lut, logits, mask_u8,
                                                                                     mask_i64, h, w);
    return e4s_launch_status();
}
