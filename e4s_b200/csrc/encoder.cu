// Elementwise / reduction kernels of the RGI encoder's conv stack (src/models/encoders/helpers.py:122-144,
// psp_encoders.py:285-309) around the tensor-core convolution (e4s_conv3x3_tcr_f32):
//   * InstanceNorm statistics per (sample, channel) -> an affine (scale, shift) that the NEXT convolution folds onto
//     its operand while staging it (no normalised tensor is ever written);
//   * the unit tail  out = 0.5 * IN(conv2) + shortcut  in one pass.  The 0.5 is the SE gate: SEModule
//     (helpers.py:56-72) gates with sigmoid(fc2(relu(fc1(mean_hw(.))))) of an InstanceNorm output, whose spatial
//     mean is zero and whose fc layers have no bias, so the gate is sigmoid(0) = 0.5 for any weights (checked
//     bit-for-bit against the oracle in tests).
// All tensors are pixel-major [B, H, W, C] fp32; these kernels are HBM/L2 streaming (the encoder's activations are
// at most 16 MB per face).
// The SPADE normalisations of face-vid2vid's generator take their statistics from a second, atomic-free pair of kernels
// (instnorm_partial_kernel, instnorm_fixed_kernel): every sum runs in an order fixed by the image size and channel count
// alone, so a sample's statistics are bit identical at any batch and on every run.
#include "common.cuh"

namespace {

constexpr int ST_WARPS = 8;

// sums[b, c, 0..1] += sum(x - k), sum((x - k)^2) with k = x[b, pixel 0, c] (shifted sums: no catastrophic cancellation)
__global__ void __launch_bounds__(32 * ST_WARPS) instnorm_stats_kernel(const float* __restrict__ x, float* __restrict__ sums,
                                                                       int hw, int c) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int b = blockIdx.z, ch = blockIdx.x * 32 + lane;
    const float* xb = x + (int64_t)b * hw * c;
    const int per = (hw + gridDim.y - 1) / gridDim.y;
    const int p0 = blockIdx.y * per, p1 = min(hw, p0 + per);
    float s1 = 0.f, s2 = 0.f;
    if (ch < c) {
        const float k = xb[ch];
        int p = p0 + warp;
        for (; p + 3 * ST_WARPS < p1; p += 4 * ST_WARPS) {       // 4 independent loads in flight per lane
            float a0 = xb[(int64_t)p * c + ch] - k, a1 = xb[(int64_t)(p + ST_WARPS) * c + ch] - k;
            float a2 = xb[(int64_t)(p + 2 * ST_WARPS) * c + ch] - k, a3 = xb[(int64_t)(p + 3 * ST_WARPS) * c + ch] - k;
            s1 += (a0 + a1) + (a2 + a3);
            s2 += (a0 * a0 + a1 * a1) + (a2 * a2 + a3 * a3);
        }
        for (; p < p1; p += ST_WARPS) {
            float a = xb[(int64_t)p * c + ch] - k;
            s1 += a, s2 += a * a;
        }
    }
    __shared__ float r1[ST_WARPS][32], r2[ST_WARPS][32];
    r1[warp][lane] = s1, r2[warp][lane] = s2;
    __syncthreads();
    if (warp == 0 && ch < c) {
        float t1 = 0.f, t2 = 0.f;
        for (int w = 0; w < ST_WARPS; ++w) t1 += r1[w][lane], t2 += r2[w][lane];
        atomicAdd(sums + ((int64_t)b * c + ch) * 2, t1);
        atomicAdd(sums + ((int64_t)b * c + ch) * 2 + 1, t2);
    }
}

// scale = rsqrt(var + eps), shift = -mean * scale   (nn.InstanceNorm2d defaults: biased variance, eps 1e-5, no affine)
__global__ void __launch_bounds__(256) instnorm_finalize_kernel(const float* __restrict__ x, const float* __restrict__ sums,
                                                                float* __restrict__ scale, float* __restrict__ shift, int batch,
                                                                int hw, int c, float eps) {
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= batch * c) return;
    const int b = i / c, ch = i - b * c;
    const float k = x[(int64_t)b * hw * c + ch];
    const float inv = 1.0f / (float)hw;
    const float m1 = sums[2 * i] * inv, m2 = sums[2 * i + 1] * inv;
    const float var = fmaxf(m2 - m1 * m1, 0.f);
    const float r = rsqrtf(var + eps);
    scale[i] = r;
    shift[i] = -(k + m1) * r;
}

// out[b,p,c] = act( alpha * (y*sy + ty) + shortcut ),  shortcut = short[b, stride*p, c] * ss + ts  (ss/ts optional)
__global__ void __launch_bounds__(256) norm_residual_kernel(const float* __restrict__ y, const float* __restrict__ sy,
                                                            const float* __restrict__ ty, float alpha,
                                                            const float* __restrict__ sh, const float* __restrict__ ss,
                                                            const float* __restrict__ ts, int sh_stride,
                                                            const float* __restrict__ slope, float* __restrict__ out, int h,
                                                            int w, int c, int64_t total4) {
    const int c4 = c >> 2;
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total4; i += (int64_t)gridDim.x * 256) {
        const int cq = (int)(i % c4);
        int64_t t = i / c4;
        const int px = (int)(t % w);
        t /= w;
        const int py = (int)(t % h);
        const int b = (int)(t / h);
        const int ch = 4 * cq;
        float4 v = *reinterpret_cast<const float4*>(y + 4 * i);
        const float4 a = __ldg(reinterpret_cast<const float4*>(sy + (int64_t)b * c + ch));
        const float4 d = __ldg(reinterpret_cast<const float4*>(ty + (int64_t)b * c + ch));
        v.x = alpha * (v.x * a.x + d.x), v.y = alpha * (v.y * a.y + d.y), v.z = alpha * (v.z * a.z + d.z), v.w = alpha * (v.w * a.w + d.w);
        if (sh) {
            const int sh_h = h * sh_stride, sh_w = w * sh_stride;
            float4 s = *reinterpret_cast<const float4*>(sh + (((int64_t)b * sh_h + (int64_t)py * sh_stride) * sh_w + (int64_t)px * sh_stride) * c + ch);
            if (ss) {
                const float4 e = __ldg(reinterpret_cast<const float4*>(ss + (int64_t)b * c + ch));
                const float4 f = __ldg(reinterpret_cast<const float4*>(ts + (int64_t)b * c + ch));
                s.x = s.x * e.x + f.x, s.y = s.y * e.y + f.y, s.z = s.z * e.z + f.z, s.w = s.w * e.w + f.w;
            }
            v.x += s.x, v.y += s.y, v.z += s.z, v.w += s.w;
        }
        if (slope) {
            const float4 q = __ldg(reinterpret_cast<const float4*>(slope + ch));
            v.x = v.x > 0.f ? v.x : v.x * q.x, v.y = v.y > 0.f ? v.y : v.y * q.y;
            v.z = v.z > 0.f ? v.z : v.z * q.z, v.w = v.w > 0.f ? v.w : v.w * q.w;
        }
        *reinterpret_cast<float4*>(out + 4 * i) = v;
    }
}

// Stage 1 of the fixed-order statistics: block (channel group, pixel block, sample) sums the IN_BLK pixels of its block
// in double, lane = channel, warp w the pixels w, w + ST_WARPS, ..; the warps' sums are added in warp order into
// part[b, blk, ch] = (sum x, sum x^2).  x pixel-pitched (pitch ld).
constexpr int IN_BLK = 1024;
__global__ void __launch_bounds__(32 * ST_WARPS) instnorm_partial_kernel(const float* __restrict__ x, int ld,
                                                                         double2* __restrict__ part, int hw, int c) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int b = blockIdx.z, blk = blockIdx.y, ch = blockIdx.x * 32 + lane;
    const int p0 = blk * IN_BLK, p1 = min(hw, p0 + IN_BLK);
    const float* xb = x + (int64_t)b * hw * ld + ch;
    double s1 = 0.0, s2 = 0.0;
    if (ch < c)
        for (int p = p0 + warp; p < p1; p += ST_WARPS) {
            const double v = __ldg(xb + (int64_t)p * ld);
            s1 += v, s2 = fma(v, v, s2);
        }
    __shared__ double r1[ST_WARPS][32], r2[ST_WARPS][32];
    r1[warp][lane] = s1, r2[warp][lane] = s2;
    __syncthreads();
    if (warp == 0 && ch < c) {
        double t1 = 0.0, t2 = 0.0;
        for (int w = 0; w < ST_WARPS; ++w) t1 += r1[w][lane], t2 += r2[w][lane];
        part[((int64_t)b * gridDim.y + blk) * c + ch] = make_double2(t1, t2);
    }
}

// Stage 2: per (sample, channel) the pixel blocks' sums in block order; mean, biased variance, scale = 1 / sqrt(var +
// eps), shift = -mean scale, in double, each rounded once to fp32
__global__ void __launch_bounds__(256) instnorm_fixed_kernel(const double2* __restrict__ part, float* __restrict__ scale,
                                                             float* __restrict__ shift, int batch, int nblk, int hw, int c,
                                                             float eps) {
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= batch * c) return;
    const int b = i / c, ch = i - b * c;
    double s1 = 0.0, s2 = 0.0;
    for (int k = 0; k < nblk; ++k) {
        const double2 v = part[((int64_t)b * nblk + k) * c + ch];
        s1 += v.x, s2 += v.y;
    }
    const double m = s1 / hw, var = fmax(s2 / hw - m * m, 0.0), r = 1.0 / sqrt(var + (double)eps);
    scale[i] = (float)r;
    shift[i] = (float)(-m * r);
}

}  // namespace

extern "C" int e4s_instnorm_stats_fixed_f32(const float* x, int x_ld, double* part_ws, float* scale, float* shift, int batch,
                                            int h, int w, int c, float eps, void* stream) {
    E4S_REQUIRE(x && part_ws && scale && shift && batch > 0 && h > 0 && w > 0 && c > 0 && x_ld >= c, E4S_ERR_ARG);
    E4S_REQUIRE(batch <= 65535 && (int64_t)h * w <= (1ll << 30), E4S_ERR_SHAPE);
    const int hw = h * w, nblk = (int)e4s_ceil_div(hw, IN_BLK);
    E4S_REQUIRE(nblk <= 65535, E4S_ERR_SHAPE);
    cudaStream_t st = (cudaStream_t)stream;
    double2* part = reinterpret_cast<double2*>(part_ws);
    instnorm_partial_kernel<<<dim3((unsigned)e4s_ceil_div(c, 32), (unsigned)nblk, (unsigned)batch), 32 * ST_WARPS, 0, st>>>(
        x, x_ld, part, hw, c);
    instnorm_fixed_kernel<<<(unsigned)e4s_ceil_div((int64_t)batch * c, 256), 256, 0, st>>>(part, scale, shift, batch, nblk, hw,
                                                                                             c, eps);
    return e4s_launch_status();
}

extern "C" int e4s_instnorm_affine_f32(const float* x, float* sums_ws, float* scale, float* shift, int batch, int h, int w,
                                       int c, float eps, void* stream) {
    E4S_REQUIRE(x && sums_ws && scale && shift && batch > 0 && h > 0 && w > 0 && c > 0, E4S_ERR_ARG);
    cudaStream_t st = (cudaStream_t)stream;
    const int hw = h * w;
    if (cudaMemsetAsync(sums_ws, 0, sizeof(float) * 2 * (size_t)batch * c, st) != cudaSuccess) return (int)cudaGetLastError();
    int chunks = (int)e4s_ceil_div(c, 32);
    int64_t want = e4s_ceil_div((int64_t)E4S_NUM_SMS * 4, (int64_t)chunks * batch);
    int splits = (int)(want < 1 ? 1 : want);
    int max_splits = (int)e4s_ceil_div(hw, 256);
    if (splits > max_splits) splits = max_splits;
    dim3 grid(chunks, splits, batch);
    instnorm_stats_kernel<<<grid, 32 * ST_WARPS, 0, st>>>(x, sums_ws, hw, c);
    instnorm_finalize_kernel<<<(unsigned)e4s_ceil_div((int64_t)batch * c, 256), 256, 0, st>>>(x, sums_ws, scale, shift, batch, hw, c, eps);
    return e4s_launch_status();
}

extern "C" int e4s_norm_residual_f32(const float* y, const float* y_scale, const float* y_shift, float alpha,
                                     const float* shortcut, const float* sc_scale, const float* sc_shift, int sc_stride,
                                     const float* prelu_slope, float* out, int batch, int h, int w, int c, void* stream) {
    E4S_REQUIRE(y && y_scale && y_shift && out && batch > 0 && h > 0 && w > 0 && c > 0, E4S_ERR_ARG);
    E4S_REQUIRE((c % 4) == 0 && (!shortcut || sc_stride == 1 || sc_stride == 2), E4S_ERR_SHAPE);
    E4S_REQUIRE((!sc_scale) == (!sc_shift), E4S_ERR_ARG);
    int64_t total4 = (int64_t)batch * h * w * (c / 4);
    int64_t want = e4s_ceil_div(total4, 256), cap = (int64_t)E4S_NUM_SMS * 16;
    norm_residual_kernel<<<(unsigned)(want < cap ? want : cap), 256, 0, (cudaStream_t)stream>>>(
        y, y_scale, y_shift, alpha, shortcut, sc_scale, sc_shift, sc_stride, prelu_slope, out, h, w, c, total4);
    return e4s_launch_status();
}
