// The small passes of face-vid2vid's keypoint detector (src/pretrained/face_vid2vid/modules/keypoint_detector.py,
// KPDetector on vox-256.yaml) around its tensor-core convolutions:
//   * input prep: AntiAliasInterpolation2d (depthwise 13 x 13 filter of the loaded buffer, zero padding 6, every 4th
//     pixel) from planar [B, 3, H, W] to the pixel-major operand [B, H / 4, W / 4, 32] of down0, channels 3..31 zero;
//   * DownBlock2d's AvgPool2d(2) after the convolution's ReLU, pixel-major;
//   * the heatmap head: per (sample, keypoint) softmax(logits / T) over the D x H x W voxels and the expectation of
//     make_coordinate_grid (x along W, y along H, z along D, each 2 i / (n - 1) - 1).
// Every sum runs in a fixed order that depends on neither the batch nor the launch: bit reproducible, batch-invariant.
#include "common.cuh"

namespace v2vkp {

constexpr int PREP_THREADS = 128, POOL_THREADS = 256, HM_THREADS = 512;
constexpr int KS = 13, PAD = 6, STEP = 4, PREP_C = 32;

// one thread per output pixel: the three channels' filter taps row-major, then the 32-channel pixel (3 values, 29 zeros)
__global__ void __launch_bounds__(PREP_THREADS) prep_kernel(const float* __restrict__ x, const float* __restrict__ wt,
                                                            float* __restrict__ y, int h, int w, int ho, int wo) {
    __shared__ float sw[3 * KS * KS];
    for (int e = threadIdx.x; e < 3 * KS * KS; e += PREP_THREADS) sw[e] = __ldg(wt + e);
    __syncthreads();
    const int ox = blockIdx.x * PREP_THREADS + threadIdx.x, oy = blockIdx.y, b = blockIdx.z;
    if (ox >= wo) return;
    float acc[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float* xc = x + ((int64_t)b * 3 + c) * h * w;
        float s = 0.f;
        for (int i = 0; i < KS; ++i) {
            const int sy = oy * STEP + i - PAD;
            if (sy < 0 || sy >= h) continue;
#pragma unroll
            for (int j = 0; j < KS; ++j) {
                const int sx = ox * STEP + j - PAD;
                if (sx >= 0 && sx < w) s = fmaf(sw[(c * KS + i) * KS + j], __ldg(xc + sy * w + sx), s);
            }
        }
        acc[c] = s;
    }
    float4* dst = reinterpret_cast<float4*>(y + (((int64_t)b * ho + oy) * wo + ox) * PREP_C);
    dst[0] = make_float4(acc[0], acc[1], acc[2], 0.f);
#pragma unroll
    for (int i = 1; i < PREP_C / 4; ++i) dst[i] = make_float4(0.f, 0.f, 0.f, 0.f);
}

// [B, H, W, C] -> [B, H / 2, W / 2, C]: (((x00 + x01) + x10) + x11) / 4, a float4 of channels per thread
__global__ void __launch_bounds__(POOL_THREADS) avgpool2_kernel(const float* __restrict__ x, float* __restrict__ y, int64_t total4,
                                                                int h, int w, int c4) {
    const int64_t i = (int64_t)blockIdx.x * POOL_THREADS + threadIdx.x;
    if (i >= total4) return;
    const int ho = h >> 1, wo = w >> 1;
    const int q = (int)(i % c4);
    int64_t r = i / c4;
    const int ox = (int)(r % wo);
    r /= wo;
    const int oy = (int)(r % ho);
    const int64_t b = r / ho;
    const float4* s = reinterpret_cast<const float4*>(x) + ((b * h + 2 * oy) * w + 2 * ox) * c4 + q;
    const float4 a = __ldg(s), bb = __ldg(s + c4), c = __ldg(s + (int64_t)w * c4), d = __ldg(s + (int64_t)w * c4 + c4);
    reinterpret_cast<float4*>(y)[i] = make_float4((((a.x + bb.x) + c.x) + d.x) / 4.f, (((a.y + bb.y) + c.y) + d.y) / 4.f,
                                                  (((a.z + bb.z) + c.z) + d.z) / 4.f, (((a.w + bb.w) + c.w) + d.w) / 4.f);
}

// fixed-order block sum of HM_THREADS values (v of every thread) -> returned to every thread; red: HM_THREADS floats
template <typename Op>
__device__ __forceinline__ float block_reduce(float v, float* red, Op op) {
    __syncthreads();
    red[threadIdx.x] = v;
    __syncthreads();
    for (int s = HM_THREADS / 2; s > 0; s >>= 1) {
        if ((int)threadIdx.x < s) red[threadIdx.x] = op(red[threadIdx.x], red[threadIdx.x + s]);
        __syncthreads();
    }
    return red[0];
}

// one CTA per (keypoint k, sample b); logits [B, H, W, D, ld] (keypoint k at channel k); voxel v = (y, x, z) in storage
// order, thread t takes v = t, t + 512, ...  Pass 1: the maximum of logit / T; pass 2: e = exp(logit / T - max), S = sum e,
// and sum e * (x, y, z); the keypoint is that sum / S.
__global__ void __launch_bounds__(HM_THREADS) heatmap_kernel(const float* __restrict__ logits, int ld, float temperature,
                                                             float* __restrict__ kp, int num_kp, int d, int h, int w) {
    __shared__ float red[HM_THREADS];
    const int k = blockIdx.x, b = blockIdx.y, t = threadIdx.x;
    const int nv = d * h * w;
    const float* src = logits + (int64_t)b * nv * ld + k;
    float m = -INFINITY;
    for (int v = t; v < nv; v += HM_THREADS) m = fmaxf(m, __ldg(src + (int64_t)v * ld) / temperature);
    m = block_reduce(m, red, [](float a, float c) { return fmaxf(a, c); });
    float s = 0.f, sx = 0.f, sy = 0.f, sz = 0.f;
    for (int v = t; v < nv; v += HM_THREADS) {
        const float e = expf(__ldg(src + (int64_t)v * ld) / temperature - m);
        const int z = v % d, x = (v / d) % w, y = v / (d * w);
        s += e;
        sx = fmaf(e, 2.f * ((float)x / (float)(w - 1)) - 1.f, sx);
        sy = fmaf(e, 2.f * ((float)y / (float)(h - 1)) - 1.f, sy);
        sz = fmaf(e, 2.f * ((float)z / (float)(d - 1)) - 1.f, sz);
    }
    auto add = [](float a, float c) { return a + c; };
    s = block_reduce(s, red, add);
    sx = block_reduce(sx, red, add);
    sy = block_reduce(sy, red, add);
    sz = block_reduce(sz, red, add);
    if (t == 0) {
        float* o = kp + ((int64_t)b * num_kp + k) * 3;
        o[0] = sx / s, o[1] = sy / s, o[2] = sz / s;
    }
}

}  // namespace v2vkp

extern "C" int e4s_vid2vid_kp_prep_f32(const float* x, const float* filter, float* y, int batch, int h, int w, void* stream) {
    E4S_REQUIRE(x && filter && y, E4S_ERR_ARG);
    E4S_REQUIRE(batch > 0 && h > 0 && w > 0 && (h % v2vkp::STEP) == 0 && (w % v2vkp::STEP) == 0, E4S_ERR_SHAPE);
    E4S_REQUIRE(e4s_aligned16(y), E4S_ERR_ALIGN);
    const int ho = h / v2vkp::STEP, wo = w / v2vkp::STEP;
    const dim3 grid((unsigned)e4s_ceil_div(wo, v2vkp::PREP_THREADS), (unsigned)ho, (unsigned)batch);
    v2vkp::prep_kernel<<<grid, v2vkp::PREP_THREADS, 0, (cudaStream_t)stream>>>(x, filter, y, h, w, ho, wo);
    return e4s_launch_status();
}

extern "C" int e4s_avgpool2_f32(const float* x, float* y, int batch, int h, int w, int c, void* stream) {
    E4S_REQUIRE(x && y, E4S_ERR_ARG);
    E4S_REQUIRE(batch > 0 && h > 1 && w > 1 && c > 0 && (h % 2) == 0 && (w % 2) == 0 && (c % 4) == 0, E4S_ERR_SHAPE);
    E4S_REQUIRE(e4s_aligned16(x) && e4s_aligned16(y), E4S_ERR_ALIGN);
    const int64_t total4 = (int64_t)batch * (h / 2) * (w / 2) * (c / 4);
    v2vkp::avgpool2_kernel<<<(unsigned)e4s_ceil_div(total4, v2vkp::POOL_THREADS), v2vkp::POOL_THREADS, 0, (cudaStream_t)stream>>>(
        x, y, total4, h, w, c / 4);
    return e4s_launch_status();
}

extern "C" int e4s_vid2vid_heatmap_f32(const float* logits, int ld, float temperature, float* kp, int batch, int num_kp, int d,
                                       int h, int w, void* stream) {
    E4S_REQUIRE(logits && kp, E4S_ERR_ARG);
    E4S_REQUIRE(batch > 0 && num_kp > 0 && num_kp <= ld && temperature > 0.f, E4S_ERR_ARG);
    E4S_REQUIRE(d > 1 && h > 1 && w > 1 && (int64_t)d * h * w * ld < (1ll << 31) && batch <= 65535, E4S_ERR_SHAPE);
    v2vkp::heatmap_kernel<<<dim3((unsigned)num_kp, (unsigned)batch), v2vkp::HM_THREADS, 0, (cudaStream_t)stream>>>(
        logits, ld, temperature, kp, num_kp, d, h, w);
    return e4s_launch_status();
}
