// Region-selected ToRGB for sm_90a: 1x1 modulated conv (no demodulation) + bias + up-sampled skip.
//
// One launch = one ToRGB.forward of the reference (src/models/stylegan2/model.py:422-448), which runs
// the 1x1 conv once per region (model.py:434-437), adds the bias (:441) and adds upfirdn2d(skip, up=2)
// (:444-446) in separate passes.  The op is a per-pixel 3 x Cin dot product: HBM-bound on reading the
// activation once (4*Cin B per pixel).  Lanes split a pixel's channels with 128-bit loads
// (pixel-major input), partial sums meet in a shuffle tree, and lanes 0..2 finish the pixel: bias,
// the 2x2 non-zero taps of the zero-stuffed 4x4 FIR on the previous RGB skip, planar store.
#include "common.cuh"

namespace {

struct TorgbParams {
    const float* x;
    const float* wrgb;
    const float* s;
    const uint8_t* label;
    const float* bias;
    const float* skip;
    const float* fir;
    float* out;
    int batch, h, w, cin, ncls;
};

// LPP = lanes per pixel (4 channels per lane per step)
template <int LPP>
__global__ void __launch_bounds__(256) torgb_kernel(TorgbParams p) {
    extern __shared__ __align__(16) float sm[];
    float* sw = sm;                       // [3][cin]
    float* ss = sm + 3 * p.cin;           // [ncls][cin]  styles of this sample
    __shared__ float sfir[16];
    const int b = blockIdx.y;
    for (int i = threadIdx.x; i < 3 * p.cin; i += 256) sw[i] = p.wrgb[i];
    for (int i = threadIdx.x; i < p.ncls * p.cin; i += 256) ss[i] = p.s[(int64_t)b * p.ncls * p.cin + i];
    if (threadIdx.x < 16) sfir[threadIdx.x] = p.fir ? p.fir[threadIdx.x] : 0.f;
    __syncthreads();

    constexpr int PPW = 32 / LPP;         // pixels per warp step
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int sub = lane / LPP, l = lane % LPP;
    const int64_t hw = (int64_t)p.h * p.w;
    const float* xb = p.x + (int64_t)b * hw * p.cin;
    const int hs = p.h / 2, ws_ = p.w / 2;

    for (int64_t pix0 = ((int64_t)blockIdx.x * 8 + warp) * PPW; pix0 < hw; pix0 += (int64_t)gridDim.x * 8 * PPW) {
        const int64_t pix = pix0 + sub;
        const bool ok = pix < hw;
        int cls = 0;
        if (ok && p.label) cls = min((int)p.label[(int64_t)b * hw + pix], p.ncls - 1);
        float a0 = 0.f, a1 = 0.f, a2 = 0.f;
        if (ok) {
            const float* xp = xb + pix * p.cin;
            const float* sp = ss + cls * p.cin;
            for (int c = 4 * l; c < p.cin; c += 4 * LPP) {
                float4 v = ld_stream_f4(xp + c);
                float4 sv = *reinterpret_cast<const float4*>(sp + c);
                v.x *= sv.x, v.y *= sv.y, v.z *= sv.z, v.w *= sv.w;
                float4 w0 = *reinterpret_cast<const float4*>(sw + c);
                float4 w1 = *reinterpret_cast<const float4*>(sw + p.cin + c);
                float4 w2 = *reinterpret_cast<const float4*>(sw + 2 * p.cin + c);
                a0 += v.x * w0.x + v.y * w0.y + v.z * w0.z + v.w * w0.w;
                a1 += v.x * w1.x + v.y * w1.y + v.z * w1.z + v.w * w1.w;
                a2 += v.x * w2.x + v.y * w2.y + v.z * w2.z + v.w * w2.w;
            }
        }
#pragma unroll
        for (int off = LPP / 2; off > 0; off >>= 1) {
            a0 += __shfl_xor_sync(0xffffffffu, a0, off);
            a1 += __shfl_xor_sync(0xffffffffu, a1, off);
            a2 += __shfl_xor_sync(0xffffffffu, a2, off);
        }
        if (ok && l < 3) {
            float v = (l == 0 ? a0 : (l == 1 ? a1 : a2)) + (p.bias ? __ldg(p.bias + l) : 0.f);
            const int yy = (int)(pix / p.w), xx = (int)(pix - (int64_t)yy * p.w);
            if (p.skip) {
                // Upsample: up=2, pad=(2,1), flipped 4x4 FIR (model.py:34-53): tap ky hits the zero-stuffed
                // grid at u = yy + ky - 2, non-zero only where u is even.
                const float* sk = p.skip + ((int64_t)b * 3 + l) * hs * ws_;
                float up = 0.f;
#pragma unroll
                for (int ky = 0; ky < 4; ++ky) {
                    int u = yy + ky - 2;
                    if (u < 0 || (u & 1) || (u >> 1) >= hs) continue;
#pragma unroll
                    for (int kx = 0; kx < 4; ++kx) {
                        int t = xx + kx - 2;
                        if (t < 0 || (t & 1) || (t >> 1) >= ws_) continue;
                        up = fmaf(__ldg(sk + (int64_t)(u >> 1) * ws_ + (t >> 1)), sfir[(3 - ky) * 4 + (3 - kx)], up);
                    }
                }
                v += up;
            }
            p.out[((int64_t)b * 3 + l) * hw + pix] = v;
        }
    }
}

// Thread-per-pixel variant for every layer whose styled weights fit 40 KB of shared memory (Cin <= 256 at 12 regions; the
// warp-per-pixel kernel above ran the 256x256 / Cin = 128 layer at 0.51 ms for 0.54 GB - one pixel per warp and iteration
// exposes the whole load -> shuffle tree -> store chain): no cross-lane reduction, weights already
// multiplied by the region's style sit in shared memory as [cls][3][cin] (broadcast reads), planar stores are
// coalesced because consecutive threads own consecutive pixels.
__global__ void __launch_bounds__(256) torgb_pixel_kernel(TorgbParams p) {
    extern __shared__ __align__(16) float sm[];
    float* ws = sm;                        // [ncls][3][cin]
    __shared__ float sfir[16];
    const int b = blockIdx.y;
    for (int i = threadIdx.x; i < p.ncls * 3 * p.cin; i += 256) {
        const int c = i / (3 * p.cin), rem = i - c * 3 * p.cin, ci = rem % p.cin;
        ws[i] = p.wrgb[rem] * p.s[((int64_t)b * p.ncls + c) * p.cin + ci];
    }
    if (threadIdx.x < 16) sfir[threadIdx.x] = p.fir ? p.fir[threadIdx.x] : 0.f;
    __syncthreads();
    const int64_t hw = (int64_t)p.h * p.w;
    const float* xb = p.x + (int64_t)b * hw * p.cin;
    const int hs = p.h / 2, ws_ = p.w / 2;
    const float b0 = p.bias ? __ldg(p.bias) : 0.f, b1 = p.bias ? __ldg(p.bias + 1) : 0.f, b2 = p.bias ? __ldg(p.bias + 2) : 0.f;
    for (int64_t pix = (int64_t)blockIdx.x * 256 + threadIdx.x; pix < hw; pix += (int64_t)gridDim.x * 256) {
        const int cls = p.label ? min((int)p.label[(int64_t)b * hw + pix], p.ncls - 1) : 0;
        const float* w0 = ws + cls * 3 * p.cin;
        const float* xp = xb + pix * p.cin;
        float a0 = b0, a1 = b1, a2 = b2;
        // a pixel's channels are one contiguous run: two adjacent 128-bit loads cover one 32-byte sector per lane
#pragma unroll 4
        for (int c = 0; c < p.cin; c += 8) {
            const float4 v = ld_stream_f4(xp + c), t = ld_stream_f4(xp + c + 4);
            const float4 u0 = *reinterpret_cast<const float4*>(w0 + c), q0 = *reinterpret_cast<const float4*>(w0 + c + 4);
            const float4 u1 = *reinterpret_cast<const float4*>(w0 + p.cin + c), q1 = *reinterpret_cast<const float4*>(w0 + p.cin + c + 4);
            const float4 u2 = *reinterpret_cast<const float4*>(w0 + 2 * p.cin + c), q2 = *reinterpret_cast<const float4*>(w0 + 2 * p.cin + c + 4);
            a0 += v.x * u0.x + v.y * u0.y + v.z * u0.z + v.w * u0.w;
            a1 += v.x * u1.x + v.y * u1.y + v.z * u1.z + v.w * u1.w;
            a2 += v.x * u2.x + v.y * u2.y + v.z * u2.z + v.w * u2.w;
            a0 += t.x * q0.x + t.y * q0.y + t.z * q0.z + t.w * q0.w;
            a1 += t.x * q1.x + t.y * q1.y + t.z * q1.z + t.w * q1.w;
            a2 += t.x * q2.x + t.y * q2.y + t.z * q2.z + t.w * q2.w;
        }
        if (p.skip) {
            const int yy = (int)(pix / p.w), xx = (int)(pix - (int64_t)yy * p.w);
            const float* sk = p.skip + (int64_t)b * 3 * hs * ws_;
#pragma unroll
            for (int ky = 0; ky < 4; ++ky) {
                const int u = yy + ky - 2;
                if (u < 0 || (u & 1) || (u >> 1) >= hs) continue;
#pragma unroll
                for (int kx = 0; kx < 4; ++kx) {
                    const int t = xx + kx - 2;
                    if (t < 0 || (t & 1) || (t >> 1) >= ws_) continue;
                    const float f = sfir[(3 - ky) * 4 + (3 - kx)];
                    const int64_t o = (int64_t)(u >> 1) * ws_ + (t >> 1);
                    a0 = fmaf(__ldg(sk + o), f, a0);
                    a1 = fmaf(__ldg(sk + (int64_t)hs * ws_ + o), f, a1);
                    a2 = fmaf(__ldg(sk + 2 * (int64_t)hs * ws_ + o), f, a2);
                }
            }
        }
        float* ob = p.out + (int64_t)b * 3 * hw + pix;
        ob[0] = a0, ob[hw] = a1, ob[2 * hw] = a2;
    }
}

template <int LPP>
int launch_torgb(const TorgbParams& p, cudaStream_t st) {
    size_t smem = sizeof(float) * (size_t)(3 + p.ncls) * p.cin;
    static E4sSmemOptIn optin;
    if (const int rc = e4s_smem_optin(optin, torgb_kernel<LPP>, smem)) return rc;
    int64_t hw = (int64_t)p.h * p.w;
    int64_t want = e4s_ceil_div(hw, 8 * (32 / LPP));
    int64_t cap = e4s_ceil_div((int64_t)E4S_NUM_SMS * 8, p.batch);   // ~8 CTAs per SM over the batch
    if (cap < 1) cap = 1;
    dim3 grid((unsigned)(want < cap ? want : cap), p.batch);
    torgb_kernel<LPP><<<grid, 256, smem, st>>>(p);
    return e4s_launch_status();
}

}  // namespace

extern "C" int e4s_torgb_fwd_f32(const float* x, const float* wrgb, const float* s, const uint8_t* label,
                                 const float* bias, const float* skip, const float* fir4x4, float* out, int batch,
                                 int h, int w, int cin, int ncls, void* stream) {
    E4S_REQUIRE(x && wrgb && s && out && batch > 0 && h > 0 && w > 0 && cin > 0 && ncls > 0, E4S_ERR_ARG);
    E4S_REQUIRE((cin % 4) == 0, E4S_ERR_SHAPE);
    E4S_REQUIRE(label || ncls == 1, E4S_ERR_ARG);
    E4S_REQUIRE(!skip || (fir4x4 && (h % 2) == 0 && (w % 2) == 0), E4S_ERR_ARG);
    E4S_REQUIRE(e4s_aligned16(x) && e4s_aligned16(s), E4S_ERR_ALIGN);
    E4S_REQUIRE((size_t)(3 + ncls) * cin * sizeof(float) <= 200 * 1024, E4S_ERR_SHAPE);
    TorgbParams p{x, wrgb, s, label, bias, skip, fir4x4, out, batch, h, w, cin, ncls};
    cudaStream_t st = (cudaStream_t)stream;
    if (cin <= 256 && (cin % 8) == 0 && (reinterpret_cast<uintptr_t>(x) & 31) == 0 &&
        (size_t)ncls * 3 * cin * sizeof(float) <= 40 * 1024) {
        const int64_t hw = (int64_t)h * w;
        int64_t want = e4s_ceil_div(hw, 256), cap = e4s_ceil_div((int64_t)E4S_NUM_SMS * 16, batch);
        if (cap < 1) cap = 1;
        dim3 grid((unsigned)(want < cap ? want : cap), batch);
        torgb_pixel_kernel<<<grid, 256, (size_t)ncls * 3 * cin * sizeof(float), st>>>(p);
        return e4s_launch_status();
    }
    if (cin >= 128) return launch_torgb<32>(p, st);
    if (cin >= 64) return launch_torgb<16>(p, st);
    if (cin >= 32) return launch_torgb<8>(p, st);
    return launch_torgb<4>(p, st);
}
