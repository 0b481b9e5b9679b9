// Kernels of the BiSeNet face parser (src/pretrained/face_parsing/) around the tensor-core convolution
// (e4s_conv3x3_bias_tcr_f32 runs every trunk, context-path and head 3x3 / 1x1 convolution):
//   * the bicubic down-sampling of FaceParser.preprocess_img (face_parsing_demo.py:15-84, 151-160) with its clamp and
//     ImageNet normalisation, in one pass;
//   * the ResNet-18 stem: 7x7 / 2 convolution (3 -> 64, BatchNorm folded) + bias + ReLU + 3x3 / 2 max-pool, fused (the
//     pre-pool map is never written);
//   * the 1x1 classifier of a BiSeNetOutput head, the bilinear (align_corners) up-sampling to the image grid and the
//     first-index argmax, with an optional 256-entry label table, in one pass;
//   * per-(sample, channel) spatial means (the attention vectors' global pooling) and the space-to-depth repack that
//     feeds a stride-2 convolution to the tensor-core kernel.
// Everything is fp32 on CUDA cores; each output is summed in a fixed order (bit reproducible, no atomics).
#include "common.cuh"

namespace parser {

__device__ __forceinline__ int reflect(int i, int n) { return i < 0 ? -i : (i >= n ? 2 * n - 2 - i : i); }

// y[b, c, oy, ox] = sum_j k[j] * t(oy, reflect(ox f - pad + j)), t(oy, x) = sum_i k[i] x[b, c, reflect(oy f - pad + i), x]
// (vertical pass first, fp32 intermediate, F.pad 'reflect'); then clamp(0, 1) and (v - mean[c]) / std[c] when mean is given.
template <int F>
__global__ void __launch_bounds__(256) bicubic_down_kernel(const float* __restrict__ x, const float* __restrict__ taps,
                                                          const float* __restrict__ mean, const float* __restrict__ std,
                                                          float* __restrict__ y, int h, int w, int64_t total) {
    constexpr int K = 4 * F, PAD = (3 * F) / 2;
    __shared__ float k[K];
    if (threadIdx.x < K) k[threadIdx.x] = taps[threadIdx.x];
    __syncthreads();
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= total) return;
    const int ho = h / F, wo = w / F;
    const int ox = (int)(i % wo), oy = (int)((i / wo) % ho);
    const int64_t plane = i / ((int64_t)wo * ho);                  // b * 3 + c
    const float* xp = x + plane * h * w;
    int rows[K];
#pragma unroll
    for (int r = 0; r < K; ++r) rows[r] = reflect(oy * F - PAD + r, h) * w;
    float acc = 0.f;
#pragma unroll
    for (int j = 0; j < K; ++j) {
        const int sx = reflect(ox * F - PAD + j, w);
        float t = 0.f;
#pragma unroll
        for (int r = 0; r < K; ++r) t = fmaf(k[r], __ldg(xp + rows[r] + sx), t);
        acc = fmaf(k[j], t, acc);
    }
    if (mean) {
        const int c = (int)(plane % 3);
        acc = (fminf(fmaxf(acc, 0.f), 1.f) - __ldg(mean + c)) / __ldg(std + c);
    }
    y[i] = acc;
}

// Stem: a CTA computes an 8 x 8 tile of pooled pixels, all 64 channels.  The 17 x 17 convolution outputs the tile's pool
// windows cover are computed from a 39 x 39 x 3 input patch in shared memory, biased, ReLU'd and kept in shared memory;
// positions outside the convolution grid hold 0, which the max over ReLU outputs (>= 0) never picks over a real value, so
// they act as the pool's -inf padding.  Thread t: channels 4 (t % 16) .. + 3 of the conv pixels t / 16 + 16 i.
constexpr int ST_PT = 8, ST_CT = 2 * ST_PT + 1, ST_IT = 2 * (ST_CT - 1) + 7;   // 8 pooled, 17 conv, 39 input
constexpr int ST_THREADS = 256;
// the patch rounded up to whole float4s, so that the weight and output tables after it are 16-byte aligned
constexpr int ST_XF = (3 * ST_IT * ST_IT + 3) & ~3;
constexpr int ST_SMEM = (ST_XF + 147 * 64 + ST_CT * ST_CT * 64) * 4;

__global__ void __launch_bounds__(ST_THREADS) stem_kernel(const float* __restrict__ x, const float* __restrict__ wt,
                                                         const float* __restrict__ bias, float* __restrict__ y, int h, int w) {
    extern __shared__ float sm[];
    float* sx = sm;                                   // [3][39][39]
    float* sw = sx + ST_XF;                           // [147][64]: tap (c, ky, kx) major, channel minor
    float* sc = sw + 147 * 64;                        // [17 * 17][64]
    const int t = threadIdx.x, b = blockIdx.z;
    const int ch = h / 2, cw = w / 2, ph = h / 4, pw = w / 4;
    const int py0 = blockIdx.y * ST_PT, px0 = blockIdx.x * ST_PT;
    const int cy0 = 2 * py0 - 1, cx0 = 2 * px0 - 1;   // first conv pixel of the tile
    const int iy0 = 2 * cy0 - 3, ix0 = 2 * cx0 - 3;   // first input pixel of the patch
    for (int e = t; e < 3 * ST_IT * ST_IT; e += ST_THREADS) {
        const int c = e / (ST_IT * ST_IT), r = (e / ST_IT) % ST_IT, q = e % ST_IT;
        const int iy = iy0 + r, ix = ix0 + q;
        sx[e] = (iy >= 0 && iy < h && ix >= 0 && ix < w) ? __ldg(x + (((int64_t)b * 3 + c) * h + iy) * w + ix) : 0.f;
    }
    for (int e = t; e < 147 * 64; e += ST_THREADS) sw[e] = __ldg(wt + (e % 64) * 147 + e / 64);
    __syncthreads();
    const int cg = (t % 16) * 4, lane_px = t / 16;
    const float4 bv = __ldg(reinterpret_cast<const float4*>(bias + cg));
    constexpr int NPIX = ST_CT * ST_CT, PER = (NPIX + 15) / 16;      // 289 conv pixels, 19 per thread at most
    constexpr int G = 4;                                              // conv pixels per pass (independent accumulators)
#pragma unroll 1
    for (int i0 = 0; i0 < PER; i0 += G) {
        float4 acc[G];
        int base[G];
#pragma unroll
        for (int g = 0; g < G; ++g) {
            acc[g] = make_float4(0.f, 0.f, 0.f, 0.f);
            const int pix = min(lane_px + 16 * (i0 + g), NPIX - 1);
            base[g] = 2 * (pix / ST_CT) * ST_IT + 2 * (pix % ST_CT);
        }
#pragma unroll 1
        for (int c = 0; c < 3; ++c)
#pragma unroll 1
            for (int ky = 0; ky < 7; ++ky)
#pragma unroll
                for (int kx = 0; kx < 7; ++kx) {
                    const int tap = (c * 7 + ky) * 7 + kx;
                    const float4 wv = *reinterpret_cast<const float4*>(sw + tap * 64 + cg);
                    const int off = (c * ST_IT + ky) * ST_IT + kx;
#pragma unroll
                    for (int g = 0; g < G; ++g) {
                        const float v = sx[base[g] + off];
                        acc[g].x = fmaf(v, wv.x, acc[g].x), acc[g].y = fmaf(v, wv.y, acc[g].y);
                        acc[g].z = fmaf(v, wv.z, acc[g].z), acc[g].w = fmaf(v, wv.w, acc[g].w);
                    }
                }
#pragma unroll
        for (int g = 0; g < G; ++g) {
            const int pix = lane_px + 16 * (i0 + g);
            if (i0 + g >= PER || pix >= NPIX) continue;
            const int cy = cy0 + pix / ST_CT, cx = cx0 + pix % ST_CT;
            float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
            if (cy >= 0 && cy < ch && cx >= 0 && cx < cw)
                o = make_float4(fmaxf(acc[g].x + bv.x, 0.f), fmaxf(acc[g].y + bv.y, 0.f), fmaxf(acc[g].z + bv.z, 0.f),
                                fmaxf(acc[g].w + bv.w, 0.f));
            *reinterpret_cast<float4*>(sc + pix * 64 + cg) = o;
        }
    }
    __syncthreads();
    // pool: 64 pooled pixels x 16 channel quads
    for (int e = t; e < ST_PT * ST_PT * 16; e += ST_THREADS) {
        const int q = e % 16, pp = e / 16, pyl = pp / ST_PT, pxl = pp % ST_PT;
        const int py = py0 + pyl, px = px0 + pxl;
        if (py >= ph || px >= pw) continue;
        float4 m = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int dy = 0; dy < 3; ++dy)
#pragma unroll
            for (int dx = 0; dx < 3; ++dx) {
                const float4 v = *reinterpret_cast<const float4*>(sc + ((2 * pyl + dy) * ST_CT + 2 * pxl + dx) * 64 + 4 * q);
                m.x = fmaxf(m.x, v.x), m.y = fmaxf(m.y, v.y), m.z = fmaxf(m.z, v.z), m.w = fmaxf(m.w, v.w);
            }
        *reinterpret_cast<float4*>(y + (((int64_t)b * ph + py) * pw + px) * 64 + 4 * q) = m;
    }
}

// Head: a CTA owns a 32 x 32 tile of the output grid.  It computes the 1x1 logits of the low-resolution pixels the tile's
// bilinear taps read (rows ly0 .. ly0 + nly - 1, columns lx0 .. + nlx - 1) into shared memory, then each thread
// interpolates its pixels (column t % 32, rows t / 32 + 8 i) class by class and keeps the first maximum.
// Source coordinate as torch's align_corners=True: s = ((in - 1) / (out - 1)) * dst in fp32, i0 = (int)s, i1 = i0 + 1 clamped,
// weight s - i0.
constexpr int HD_T = 32, HD_THREADS = 256;

__device__ __forceinline__ float src_scale(int in, int out) { return out > 1 ? (float)(in - 1) / (float)(out - 1) : 0.f; }

__global__ void __launch_bounds__(HD_THREADS) head_kernel(const float* __restrict__ x, const float* __restrict__ wt,
                                                         const uint8_t* __restrict__ lut, uint8_t* __restrict__ labels,
                                                         float* __restrict__ logits, int h, int w, int c, int ncls, int oh,
                                                         int ow, int max_rows, int max_cols) {
    extern __shared__ float sm[];
    float* sw = sm;                                       // [ncls][c]
    float* sl = sw + ncls * c;                            // [max_rows][max_cols][ncls]
    const int t = threadIdx.x, b = blockIdx.z;
    const int Y0 = blockIdx.y * HD_T, X0 = blockIdx.x * HD_T;
    const float shy = src_scale(h, oh), shx = src_scale(w, ow);
    const int ly0 = (int)(shy * (float)Y0), lx0 = (int)(shx * (float)X0);
    const int ly1 = min((int)(shy * (float)min(Y0 + HD_T - 1, oh - 1)) + 1, h - 1);
    const int lx1 = min((int)(shx * (float)min(X0 + HD_T - 1, ow - 1)) + 1, w - 1);
    const int nly = ly1 - ly0 + 1, nlx = lx1 - lx0 + 1;
    for (int e = t; e < ncls * c; e += HD_THREADS) sw[e] = __ldg(wt + e);
    __syncthreads();
    const int c4 = c / 4;
    for (int e = t; e < nly * nlx * ncls; e += HD_THREADS) {
        const int k = e % ncls, pix = e / ncls, ly = ly0 + pix / nlx, lx = lx0 + pix % nlx;
        const float4* xv = reinterpret_cast<const float4*>(x + (((int64_t)b * h + ly) * w + lx) * c);
        const float4* wv = reinterpret_cast<const float4*>(sw + k * c);
        float a = 0.f;
        for (int q = 0; q < c4; ++q) {
            const float4 u = __ldg(xv + q), v = wv[q];
            a = fmaf(u.x, v.x, a), a = fmaf(u.y, v.y, a), a = fmaf(u.z, v.z, a), a = fmaf(u.w, v.w, a);
        }
        sl[((pix / nlx) * max_cols + pix % nlx) * ncls + k] = a;
    }
    __syncthreads();
    const int X = X0 + (t % HD_T);
    if (X >= ow) return;
    const float sx = shx * (float)X;
    const int x0 = (int)sx, x1 = x0 + (x0 < w - 1 ? 1 : 0);
    const float fx1 = sx - (float)x0, fx0 = 1.f - fx1;
    for (int Y = Y0 + t / HD_T; Y < min(Y0 + HD_T, oh); Y += HD_THREADS / HD_T) {
        const float sy = shy * (float)Y;
        const int y0 = (int)sy, y1 = y0 + (y0 < h - 1 ? 1 : 0);
        const float fy1 = sy - (float)y0, fy0 = 1.f - fy1;
        const float* p00 = sl + ((y0 - ly0) * max_cols + (x0 - lx0)) * ncls;
        const float* p01 = sl + ((y0 - ly0) * max_cols + (x1 - lx0)) * ncls;
        const float* p10 = sl + ((y1 - ly0) * max_cols + (x0 - lx0)) * ncls;
        const float* p11 = sl + ((y1 - ly0) * max_cols + (x1 - lx0)) * ncls;
        float best = 0.f;
        int arg = 0;
        for (int k = 0; k < ncls; ++k) {
            const float v = fy0 * (fx0 * p00[k] + fx1 * p01[k]) + fy1 * (fx0 * p10[k] + fx1 * p11[k]);
            if (logits) logits[(((int64_t)b * ncls + k) * oh + Y) * ow + X] = v;
            if (k == 0 || v > best) best = v, arg = k;
        }
        if (labels) labels[((int64_t)b * oh + Y) * ow + X] = lut ? __ldg(lut + arg) : (uint8_t)arg;
    }
}

// y[b, c] = mean over the hw pixels of pixel-major x[b, :, c].  A CTA per (sample, 32 channels): warp v sums pixels
// v, v + 8, ... in order, then warp 0 adds the eight partial sums in order.
constexpr int MN_WARPS = 8;
__global__ void __launch_bounds__(32 * MN_WARPS) channel_mean_kernel(const float* __restrict__ x, float* __restrict__ y, int hw,
                                                                     int c) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int b = blockIdx.y, ch = blockIdx.x * 32 + lane;
    __shared__ float part[MN_WARPS][32];
    float s = 0.f;
    if (ch < c)
        for (int p = warp; p < hw; p += MN_WARPS) s += __ldg(x + ((int64_t)b * hw + p) * c + ch);
    part[warp][lane] = s;
    __syncthreads();
    if (warp == 0 && ch < c) {
        float tot = 0.f;
        for (int v = 0; v < MN_WARPS; ++v) tot += part[v][lane];
        y[(int64_t)b * c + ch] = tot / (float)hw;
    }
}

// y[b, i, j, (py * 2 + px) * c + ch] = x[b, 2 i + py, 2 j + px, ch], float4 per thread
__global__ void __launch_bounds__(256) space_to_depth_kernel(const float* __restrict__ x, float* __restrict__ y, int h, int w,
                                                             int c, int64_t total4) {
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= total4) return;
    const int c4 = c / 4;
    const int q = (int)(i % c4);
    int64_t r = i / c4;
    const int px = (int)(r % w);
    r /= w;
    const int py = (int)(r % h);
    const int b = (int)(r / h);
    const float4 v = ld_stream_f4(x + 4 * i);
    const int ho = h / 2, wo = w / 2;
    float* dst = y + (((int64_t)b * ho + (py >> 1)) * wo + (px >> 1)) * 4 * c + ((py & 1) * 2 + (px & 1)) * c + 4 * q;
    *reinterpret_cast<float4*>(dst) = v;
}

}  // namespace parser

extern "C" int e4s_bicubic_down_norm_f32(const float* x, const float* taps, const float* mean, const float* std, float* y,
                                         int batch, int h, int w, int factor, void* stream) {
    E4S_REQUIRE(x && taps && y && batch > 0 && (!mean) == (!std), E4S_ERR_ARG);
    E4S_REQUIRE((factor == 1 || factor == 2 || factor == 4) && h % factor == 0 && w % factor == 0 && h >= 4 * factor &&
                    w >= 4 * factor,
                E4S_ERR_SHAPE);
    const int64_t total = (int64_t)batch * 3 * (h / factor) * (w / factor);
    const unsigned blocks = (unsigned)e4s_ceil_div(total, 256);
    cudaStream_t st = (cudaStream_t)stream;
    if (factor == 1) parser::bicubic_down_kernel<1><<<blocks, 256, 0, st>>>(x, taps, mean, std, y, h, w, total);
    else if (factor == 2) parser::bicubic_down_kernel<2><<<blocks, 256, 0, st>>>(x, taps, mean, std, y, h, w, total);
    else parser::bicubic_down_kernel<4><<<blocks, 256, 0, st>>>(x, taps, mean, std, y, h, w, total);
    return e4s_launch_status();
}

extern "C" int e4s_parser_stem_f32(const float* x, const float* w7x7, const float* bias, float* y, int batch, int h, int w,
                                   void* stream) {
    E4S_REQUIRE(x && w7x7 && bias && y && batch > 0 && h > 0 && w > 0, E4S_ERR_ARG);
    E4S_REQUIRE(h % 4 == 0 && w % 4 == 0 && batch < 65536, E4S_ERR_SHAPE);
    E4S_REQUIRE(e4s_aligned16(bias) && e4s_aligned16(y), E4S_ERR_ALIGN);
    static E4sSmemOptIn optin;
    if (const int rc = e4s_smem_optin(optin, parser::stem_kernel, parser::ST_SMEM)) return rc;
    dim3 grid((unsigned)e4s_ceil_div(w / 4, parser::ST_PT), (unsigned)e4s_ceil_div(h / 4, parser::ST_PT), batch);
    parser::stem_kernel<<<grid, parser::ST_THREADS, parser::ST_SMEM, (cudaStream_t)stream>>>(x, w7x7, bias, y, h, w);
    return e4s_launch_status();
}

extern "C" int e4s_parse_head_u8(const float* x, const float* w1x1, const uint8_t* lut, uint8_t* labels, float* logits,
                                 int batch, int h, int w, int c, int ncls, int out_h, int out_w, void* stream) {
    E4S_REQUIRE(x && w1x1 && (labels || logits) && batch > 0 && h > 0 && w > 0 && c > 0, E4S_ERR_ARG);
    E4S_REQUIRE(ncls > 0 && ncls <= 32 && c % 4 == 0 && out_h >= h && out_w >= w && batch < 65536, E4S_ERR_SHAPE);
    E4S_REQUIRE(e4s_aligned16(x) && e4s_aligned16(w1x1), E4S_ERR_ALIGN);
    // low-resolution rows / columns one 32-pixel tile reads: floor(s Y1) - floor(s Y0) + 2 <= floor(31 s) + 3 with
    // s = (in - 1) / (out - 1), plus one for the fp32 rounding of s Y
    const int max_rows = (out_h > 1 ? (parser::HD_T - 1) * (h - 1) / (out_h - 1) : 0) + 4;
    const int max_cols = (out_w > 1 ? (parser::HD_T - 1) * (w - 1) / (out_w - 1) : 0) + 4;
    const size_t smem = sizeof(float) * ((size_t)ncls * c + (size_t)max_rows * max_cols * ncls);
    E4S_REQUIRE(smem <= (size_t)e4s_smem_optin_limit(), E4S_ERR_SHAPE);
    static E4sSmemOptIn optin;
    if (const int rc = e4s_smem_optin(optin, parser::head_kernel, smem)) return rc;
    dim3 grid((unsigned)e4s_ceil_div(out_w, parser::HD_T), (unsigned)e4s_ceil_div(out_h, parser::HD_T), batch);
    parser::head_kernel<<<grid, parser::HD_THREADS, smem, (cudaStream_t)stream>>>(x, w1x1, lut, labels, logits, h, w, c, ncls,
                                                                                  out_h, out_w, max_rows, max_cols);
    return e4s_launch_status();
}

extern "C" int e4s_channel_mean_f32(const float* x, float* y, int batch, int hw, int c, void* stream) {
    E4S_REQUIRE(x && y && batch > 0 && hw > 0 && c > 0, E4S_ERR_ARG);
    E4S_REQUIRE(batch < 65536, E4S_ERR_SHAPE);
    dim3 grid((unsigned)e4s_ceil_div(c, 32), batch);
    parser::channel_mean_kernel<<<grid, 32 * parser::MN_WARPS, 0, (cudaStream_t)stream>>>(x, y, hw, c);
    return e4s_launch_status();
}

extern "C" int e4s_space_to_depth_f32(const float* x, float* y, int batch, int h, int w, int c, void* stream) {
    E4S_REQUIRE(x && y && batch > 0 && h > 0 && w > 0 && c > 0, E4S_ERR_ARG);
    E4S_REQUIRE(h % 2 == 0 && w % 2 == 0 && c % 4 == 0, E4S_ERR_SHAPE);
    E4S_REQUIRE(e4s_aligned16(x) && e4s_aligned16(y), E4S_ERR_ALIGN);
    const int64_t total4 = (int64_t)batch * h * w * (c / 4);
    parser::space_to_depth_kernel<<<(unsigned)e4s_ceil_div(total4, 256), 256, 0, (cudaStream_t)stream>>>(x, y, h, w, c, total4);
    return e4s_launch_status();
}
