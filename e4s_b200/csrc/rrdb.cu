// The RGB-side convolutions of ESRGAN's RRDBNet (src/pretrained/gpen/sr_model/rrdbnet_arch.py): conv_first (3 -> 32
// channels, planar image in, pixel-major features out) and conv_last (32 -> 3, pixel-major features in, planar image out),
// both 3x3, stride 1, padding 1, + bias.  They are 0.15 % of the network's multiply-adds; every other convolution of it runs
// on the tensor-core kernel (e4s_conv3x3_dense_tcr_f32).  fp32 on CUDA cores: a thread computes every output channel of one
// pixel, the 27 / 288 input values it needs read once, the weights from shared memory (a broadcast: every thread of a warp
// reads the same word).  Each output sums taps row-major, channels ascending, then adds the bias (bit reproducible).
#include "common.cuh"

namespace rrdb {

constexpr int RGB_THREADS = 128;      // pixels of one image row per CTA

// CIN 3 / COUT 32: x planar [B, 3, H, W], y pixel-major with pitch y_ld; CIN 32 / COUT 3: x pixel-major with pitch x_ld,
// y planar [B, 3, H, W].  w: nn.Conv2d layout [COUT][CIN][3][3]; bias [COUT].
template <int CIN, int COUT>
__global__ void __launch_bounds__(RGB_THREADS) conv3x3_rgb_kernel(const float* __restrict__ x, int x_ld, const float* __restrict__ wt,
                                                                  const float* __restrict__ bias, float* __restrict__ y, int y_ld,
                                                                  int h, int w) {
    constexpr bool PLANAR_IN = CIN == 3;
    // [tap][ci][co] for the planar input (a pixel's value times COUT consecutive weights), [tap][co][ci] for the
    // pixel-major one (float4 weight reads along the channels)
    __shared__ __align__(16) float sw[9 * CIN * COUT];
    __shared__ float sb[COUT];
    for (int e = threadIdx.x; e < 9 * CIN * COUT; e += RGB_THREADS) {
        const int tap = e / (COUT * CIN);
        const int co = PLANAR_IN ? e % COUT : (e / CIN) % COUT, ci = PLANAR_IN ? (e / COUT) % CIN : e % CIN;
        sw[e] = __ldg(wt + (co * CIN + ci) * 9 + tap);
    }
    if (threadIdx.x < COUT) sb[threadIdx.x] = __ldg(bias + threadIdx.x);
    __syncthreads();
    const int ox = blockIdx.x * RGB_THREADS + threadIdx.x, oy = blockIdx.y, b = blockIdx.z;
    if (ox >= w) return;
    float acc[COUT];
#pragma unroll
    for (int co = 0; co < COUT; ++co) acc[co] = 0.f;
#pragma unroll
    for (int tap = 0; tap < 9; ++tap) {
        const int sy = oy + tap / 3 - 1, sx = ox + tap % 3 - 1;
        if (sy < 0 || sy >= h || sx < 0 || sx >= w) continue;
        if constexpr (PLANAR_IN) {
#pragma unroll
            for (int ci = 0; ci < CIN; ++ci) {
                const float v = __ldg(x + (((int64_t)b * CIN + ci) * h + sy) * w + sx);
                const float* wr = sw + (tap * CIN + ci) * COUT;
#pragma unroll
                for (int co = 0; co < COUT; ++co) acc[co] = fmaf(v, wr[co], acc[co]);
            }
        } else {
            const float* xp = x + (((int64_t)b * h + sy) * w + sx) * x_ld;
#pragma unroll
            for (int c4 = 0; c4 < CIN / 4; ++c4) {
                const float4 v = __ldg(reinterpret_cast<const float4*>(xp) + c4);
#pragma unroll
                for (int co = 0; co < COUT; ++co) {
                    const float4 wv = *reinterpret_cast<const float4*>(sw + (tap * COUT + co) * CIN + 4 * c4);
                    acc[co] = fmaf(v.w, wv.w, fmaf(v.z, wv.z, fmaf(v.y, wv.y, fmaf(v.x, wv.x, acc[co]))));
                }
            }
        }
    }
    if constexpr (PLANAR_IN) {
        float* yp = y + (((int64_t)b * h + oy) * w + ox) * y_ld;
#pragma unroll
        for (int c4 = 0; c4 < COUT / 4; ++c4)
            reinterpret_cast<float4*>(yp)[c4] = make_float4(acc[4 * c4] + sb[4 * c4], acc[4 * c4 + 1] + sb[4 * c4 + 1],
                                                            acc[4 * c4 + 2] + sb[4 * c4 + 2], acc[4 * c4 + 3] + sb[4 * c4 + 3]);
    } else {
#pragma unroll
        for (int co = 0; co < COUT; ++co) y[(((int64_t)b * COUT + co) * h + oy) * w + ox] = acc[co] + sb[co];
    }
}

}  // namespace rrdb

extern "C" int e4s_conv3x3_rgb_f32(const float* x, int x_ld, const float* w3x3, const float* bias, float* y, int y_ld, int batch,
                                   int h, int w, int cin, int cout, void* stream) {
    E4S_REQUIRE(x && w3x3 && bias && y && batch > 0 && h > 0 && w > 0, E4S_ERR_ARG);
    E4S_REQUIRE(((cin == 3 && cout == 32) || (cin == 32 && cout == 3)) && batch < 65536 && h < 65536, E4S_ERR_SHAPE);
    E4S_REQUIRE(cin == 3 ? y_ld >= cout : x_ld >= cin, E4S_ERR_ARG);
    E4S_REQUIRE((cin == 3 ? y_ld % 4 == 0 && e4s_aligned16(y) : x_ld % 4 == 0 && e4s_aligned16(x)), E4S_ERR_ALIGN);
    const dim3 grid((unsigned)e4s_ceil_div(w, rrdb::RGB_THREADS), (unsigned)h, (unsigned)batch);
    cudaStream_t st = (cudaStream_t)stream;
    if (cin == 3)
        rrdb::conv3x3_rgb_kernel<3, 32><<<grid, rrdb::RGB_THREADS, 0, st>>>(x, x_ld, w3x3, bias, y, y_ld, h, w);
    else
        rrdb::conv3x3_rgb_kernel<32, 3><<<grid, rrdb::RGB_THREADS, 0, st>>>(x, x_ld, w3x3, bias, y, y_ld, h, w);
    return e4s_launch_status();
}
