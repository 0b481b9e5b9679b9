// Fused bias + leaky-ReLU (+ gradient) for sm_90a.
//
// Replaces fused_bias_act_kernel of the reference (fused_bias_act_kernel.cu:18-49: 128 threads,
// 4 scalar elements per thread).  Pure HBM streaming: 128-bit loads/stores, grid-stride over a grid
// sized in waves of the 132 SMs.  In the synthesis network this op is normally folded into the
// convolution epilogue (modconv); the standalone entry points serve the op-level API
// (fused_leaky_relu / FusedLeakyReLU, fused_act.py:72-85) and the mapping network's EqualLinear.
#include "common.cuh"

namespace {

__global__ void __launch_bounds__(256) bias_act_fwd_kernel(const float* __restrict__ x, const float* __restrict__ bias,
                                                           float* __restrict__ y, int64_t n, int step_b, int size_b,
                                                           float alpha, float scale, bool vec) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (vec) {
        // step_b % 4 == 0 (or step_b == 1 with size_b % 4 == 0): a float4 never straddles... see host code
        const int64_t n4 = n >> 2;
        for (; i < n4; i += stride) {
            float4 v = ld_stream_f4(x + 4 * i);
            int64_t e = 4 * i;
            if (bias) {
                if (step_b == 1) {
                    int c = (int)(e % size_b);
                    v.x += __ldg(bias + c), v.y += __ldg(bias + c + 1), v.z += __ldg(bias + c + 2), v.w += __ldg(bias + c + 3);
                } else {
                    float b = __ldg(bias + (int)((e / step_b) % size_b));
                    v.x += b, v.y += b, v.z += b, v.w += b;
                }
            }
            v.x = lrelu_scaled(v.x, alpha, scale), v.y = lrelu_scaled(v.y, alpha, scale);
            v.z = lrelu_scaled(v.z, alpha, scale), v.w = lrelu_scaled(v.w, alpha, scale);
            st_stream_f4(y + 4 * i, v);
        }
    } else {
        for (; i < n; i += stride) {
            float v = x[i];
            if (bias) v += __ldg(bias + (int)((i / step_b) % size_b));
            y[i] = lrelu_scaled(v, alpha, scale);
        }
    }
}

__global__ void __launch_bounds__(256) bias_act_bwd_kernel(const float* __restrict__ g, const float* __restrict__ ref,
                                                           float* __restrict__ gx, int64_t n, float alpha, float scale,
                                                           bool vec) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (vec) {
        const int64_t n4 = n >> 2;
        for (; i < n4; i += stride) {
            float4 a = ld_stream_f4(g + 4 * i), r = ld_stream_f4(ref + 4 * i);
            a.x = (r.x > 0.f ? a.x : a.x * alpha) * scale;
            a.y = (r.y > 0.f ? a.y : a.y * alpha) * scale;
            a.z = (r.z > 0.f ? a.z : a.z * alpha) * scale;
            a.w = (r.w > 0.f ? a.w : a.w * alpha) * scale;
            st_stream_f4(gx + 4 * i, a);
        }
    } else {
        for (; i < n; i += stride) gx[i] = (ref[i] > 0.f ? g[i] : g[i] * alpha) * scale;
    }
}

// gb[c] = sum over outer, step of gx[outer, c, step].  One CTA per channel slice; deterministic
// (fixed reduction order, no atomics).
__global__ void __launch_bounds__(256) bias_grad_kernel(const float* __restrict__ gx, float* __restrict__ gb,
                                                        int64_t outer, int size_b, int step_b) {
    const int c = blockIdx.x;
    float acc = 0.f;
    if (step_b == 1) {
        for (int64_t o = threadIdx.x; o < outer; o += blockDim.x) acc += gx[o * size_b + c];
    } else {
        const int64_t per = (int64_t)outer * step_b;
        for (int64_t e = threadIdx.x; e < per; e += blockDim.x) {
            int64_t o = e / step_b;
            int s = (int)(e - o * step_b);
            acc += gx[(o * size_b + c) * step_b + s];
        }
    }
    __shared__ float red[256];
    red[threadIdx.x] = acc;
    __syncthreads();
    for (int s = 128; s > 0; s >>= 1) {
        if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
        __syncthreads();
    }
    if (threadIdx.x == 0) gb[c] = red[0];
}

inline unsigned stream_grid(int64_t work_items) {
    int64_t want = e4s_ceil_div(work_items, 256);
    int64_t cap = (int64_t)E4S_NUM_SMS * 16;
    if (want < 1) want = 1;
    return (unsigned)(want < cap ? want : cap);
}

}  // namespace

extern "C" int e4s_bias_act_fwd_f32(const float* x, const float* bias, float* y, int64_t n, int step_b, int size_b,
                                    float alpha, float scale, void* stream) {
    E4S_REQUIRE(x && y && n >= 0, E4S_ERR_ARG);
    if (n == 0) return E4S_OK;
    if (bias) E4S_REQUIRE(step_b > 0 && size_b > 0, E4S_ERR_ARG);
    if (!bias) step_b = 1, size_b = 1;
    // 128-bit path when a float4 stays inside one bias run (planar) or one pixel's channels (pixel-major)
    bool vec = (n % 4 == 0) && e4s_aligned16(x) && e4s_aligned16(y) &&
               (!bias || (step_b % 4 == 0) || (step_b == 1 && size_b % 4 == 0));
    bias_act_fwd_kernel<<<stream_grid(vec ? n / 4 : n), 256, 0, (cudaStream_t)stream>>>(x, bias, y, n, step_b, size_b,
                                                                                          alpha, scale, vec);
    return e4s_launch_status();
}

extern "C" int e4s_bias_act_bwd_f32(const float* g, const float* ref, float* gx, int64_t n, float alpha, float scale,
                                    void* stream) {
    E4S_REQUIRE(g && ref && gx && n >= 0, E4S_ERR_ARG);
    if (n == 0) return E4S_OK;
    bool vec = (n % 4 == 0) && e4s_aligned16(g) && e4s_aligned16(ref) && e4s_aligned16(gx);
    bias_act_bwd_kernel<<<stream_grid(vec ? n / 4 : n), 256, 0, (cudaStream_t)stream>>>(g, ref, gx, n, alpha, scale, vec);
    return e4s_launch_status();
}

extern "C" int e4s_bias_grad_f32(const float* gx, float* gb, int64_t outer, int size_b, int step_b, void* stream) {
    E4S_REQUIRE(gx && gb && outer > 0 && size_b > 0 && step_b > 0, E4S_ERR_ARG);
    bias_grad_kernel<<<size_b, 256, 0, (cudaStream_t)stream>>>(gx, gb, outer, size_b, step_b);
    return e4s_launch_status();
}
