// Backward of the fused StyledConv / ToRGB ops (sm_90a, fp32 SIMT): input- and style-gradients.
//
// The reference's inversion loop (scripts/optimization.py:209-232) back-propagates through the generator with
// autograd: per region per layer one cuDNN dgrad AND one wgrad (the per-sample modulated weight carries the
// style's gradient, src/models/stylegan2/model.py:277), plus the elementwise chain.  With the shared-weight form
//     u[p,o] = sum_{i,k} W[k][i][o] s[c(p),i] x[p+k,i],   v = u d[c(p),o] + w_n n[p] + b[o],   y = act(v)
// the weights are constants (frozen, networks.py:69-71) and the whole backward is
//     gv = act'(y) gy
//     G_c[q,i] = sum_{o,k} W[8-k][i][o] * ( gv[q+k-1,o] d[c,o] [c(q+k-1) == c] )         one dgrad conv per region present
//     gx[q,i]  = sum_c s[c,i] G_c[q,i]
//     gs[c,i]  = sum_q x[q,i] G_c[q,i]   -   s[c,i] sum_o gdu[c,o] d[c,o]^2 Wsq[o,i]       (conv path + demod path)
//     gdu[c,o] = sum_{p in c} gv[p,o] (v[p,o] - w_n n[p] - b[o])
// i.e. style gradients are REDUCTIONS in the dgrad epilogue - no per-sample weight-gradient GEMM exists.
// Up-sampling layers: the forward is four parity convs on the input grid, so the dgrad sums four parity planes
// of gy (stride-2 gathers) against the spatially flipped folded kernels.
//
// Kernels here:
//   modconv3x3_dgrad_kernel  - G_c, gx and the conv-path part of gs (atomics into [B, ncls, Cin])
//   class_reduce_kernel      - gdu[b,c,o] (and optionally the noise gradient)
//   torgb_bwd_kernel         - gx, gs of the 1x1 ToRGB conv
#include "common.cuh"

namespace {

constexpr int KC = 16;
constexpr int TH = 8;
constexpr int MAXCLS = 32;
constexpr float SQRT2 = 1.41421356237309515f;

struct DgradParams {
    const float* gy;       // [B, Ho, Wo, Cout]
    const float* y;        // forward output (for act'), or NULL when act == 0
    const float* x;        // [B, H, W, Cin] forward input (style gradient), or NULL
    const float* wd;       // [nphase][9][Cout][Cin], taps already flipped
    const float* s;        // [B, ncls, Cin]
    const float* demod;    // [B, ncls, Cout] or NULL
    const uint8_t* label;  // [B, Ho, Wo] or NULL
    float* gx;             // [B, H, W, Cin] or NULL
    float* gs;             // [B, ncls, Cin] accumulated atomically, or NULL
    int batch, h, w, cin, cout, ncls, up, act;
    int tiles_x, tiles_y;
};

template <int ICG>
__global__ void __launch_bounds__(256) modconv3x3_dgrad_kernel(DgradParams p) {
    constexpr int PG = 256 / ICG;
    constexpr int TW = 4 * PG / TH;
    constexpr int XW = TW + 4;
    constexpr int XR = TH + 2;
    constexpr int ICT = 4 * ICG;           // input channels (outputs of the dgrad) per tile
    constexpr int XS_O = XR * XW;

    extern __shared__ __align__(16) float smem[];
    float* gsm = smem;                      // [KC][XR][XW]   staged, transformed gy
    float* ws = gsm + KC * XS_O;            // [KC][9][ICT]
    float* red = ws + KC * 9 * ICT;         // [PG][ICT] style-gradient partials
    __shared__ unsigned cls_mask;

    int bid = blockIdx.x;
    const int tile_x = bid % p.tiles_x;
    bid /= p.tiles_x;
    const int tile_y = bid % p.tiles_y;
    const int b = bid / p.tiles_y;
    const int i0 = blockIdx.y * ICT;
    const int nphase = p.up ? 4 : 1;
    const int mul = p.up ? 2 : 1;
    const int ho = p.h * mul, wo = p.w * mul;

    const int ig = threadIdx.x % ICG, pg = threadIdx.x / ICG;
    const int prow = pg / (TW / 4), pcol = 4 * (pg % (TW / 4));
    const int qy = tile_y * TH + prow, qx0 = tile_x * TW + pcol;
    const int y_in0 = tile_y * TH - 1, x_in0 = tile_x * TW - 1;

    // ---- regions present among the source pixels (halo, all parities)
    if (threadIdx.x == 0) cls_mask = p.label ? 0u : 1u;
    __syncthreads();
    if (p.label) {
        unsigned m = 0;
        for (int e = threadIdx.x; e < XR * (TW + 2) * nphase; e += 256) {
            int ph = e % nphase, pix = e / nphase;
            int r = pix / (TW + 2), c = pix - r * (TW + 2);
            int gyy = y_in0 + r, gxx = x_in0 + c;
            if (gyy >= 0 && gyy < p.h && gxx >= 0 && gxx < p.w) {
                int cl = p.label[((int64_t)b * ho + gyy * mul + (ph >> 1)) * wo + gxx * mul + (ph & 1)];
                m |= 1u << min(cl, p.ncls - 1);
            }
        }
        if (m) atomicOr(&cls_mask, m);
    }
    __syncthreads();
    const unsigned classes = cls_mask;

    bool valid[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) valid[q] = (qy < p.h) && (qx0 + q < p.w);
    const int ci = i0 + 4 * ig;
    const bool ci_ok = ci < p.cin;

    float gxacc[4][4];
#pragma unroll
    for (int q = 0; q < 4; ++q)
#pragma unroll
        for (int i = 0; i < 4; ++i) gxacc[q][i] = 0.f;

    const float* gyb = p.gy + (int64_t)b * ho * wo * p.cout;
    const float* yb = p.y ? p.y + (int64_t)b * ho * wo * p.cout : nullptr;

    for (unsigned cm = classes; cm; cm &= cm - 1) {
        const int cls = __ffs(cm) - 1;
        float acc[4][4];
#pragma unroll
        for (int q = 0; q < 4; ++q)
#pragma unroll
            for (int i = 0; i < 4; ++i) acc[q][i] = 0.f;
        const float* dmc = p.demod ? p.demod + ((int64_t)b * p.ncls + cls) * p.cout : nullptr;

        for (int ph = 0; ph < nphase; ++ph) {
            const int py = ph >> 1, px = ph & 1;
            const float* wph = p.wd + (int64_t)ph * 9 * p.cout * p.cin;
            for (int o0 = 0; o0 < p.cout; o0 += KC) {
                __syncthreads();
                // stage the class-masked, activation- and demod-scaled output gradient of this parity plane
                for (int e = threadIdx.x; e < XR * (TW + 2) * (KC / 4); e += 256) {
                    int oq = e % (KC / 4);
                    int pix = e / (KC / 4);
                    int r = pix / (TW + 2), c = pix - r * (TW + 2);
                    int sy = y_in0 + r, sx = x_in0 + c, o = o0 + 4 * oq;
                    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (sy >= 0 && sy < p.h && sx >= 0 && sx < p.w && o < p.cout) {
                        const int oy = sy * mul + py, ox = sx * mul + px;
                        const int cl = p.label ? min((int)p.label[((int64_t)b * ho + oy) * wo + ox], p.ncls - 1) : 0;
                        if (cl == cls) {
                            const int64_t off = ((int64_t)oy * wo + ox) * p.cout + o;
                            v = *reinterpret_cast<const float4*>(gyb + off);
                            if (p.act) {
                                float4 yv = *reinterpret_cast<const float4*>(yb + off);
                                v.x *= yv.x > 0.f ? SQRT2 : 0.2f * SQRT2;
                                v.y *= yv.y > 0.f ? SQRT2 : 0.2f * SQRT2;
                                v.z *= yv.z > 0.f ? SQRT2 : 0.2f * SQRT2;
                                v.w *= yv.w > 0.f ? SQRT2 : 0.2f * SQRT2;
                            }
                            if (dmc) {
                                float4 d = __ldg(reinterpret_cast<const float4*>(dmc + o));
                                v.x *= d.x, v.y *= d.y, v.z *= d.z, v.w *= d.w;
                            }
                        }
                    }
                    float* dst = gsm + (4 * oq) * XS_O + r * XW + c;
                    dst[0] = v.x, dst[XS_O] = v.y, dst[2 * XS_O] = v.z, dst[3 * XS_O] = v.w;
                }
                for (int e = threadIdx.x; e < KC * 9 * ICG; e += 256) {
                    int c4 = e % ICG;
                    int t = e / ICG;
                    int tap = t % 9, o = t / 9;
                    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                    int cc = i0 + 4 * c4;
                    if (o0 + o < p.cout && cc < p.cin)
                        v = __ldg(reinterpret_cast<const float4*>(wph + ((int64_t)tap * p.cout + o0 + o) * p.cin + cc));
                    *reinterpret_cast<float4*>(ws + (o * 9 + tap) * ICT + 4 * c4) = v;
                }
                __syncthreads();
#pragma unroll 4
                for (int o = 0; o < KC; ++o) {
#pragma unroll
                    for (int dy = 0; dy < 3; ++dy) {
                        const float* xr = gsm + o * XS_O + (prow + dy) * XW + pcol;
                        float4 a = *reinterpret_cast<const float4*>(xr);
                        float2 c2 = *reinterpret_cast<const float2*>(xr + 4);
                        float xv[6] = {a.x, a.y, a.z, a.w, c2.x, c2.y};
#pragma unroll
                        for (int dx = 0; dx < 3; ++dx) {
                            float4 wv = *reinterpret_cast<const float4*>(ws + (o * 9 + dy * 3 + dx) * ICT + 4 * ig);
#pragma unroll
                            for (int q = 0; q < 4; ++q) {
                                acc[q][0] = fmaf(xv[q + dx], wv.x, acc[q][0]);
                                acc[q][1] = fmaf(xv[q + dx], wv.y, acc[q][1]);
                                acc[q][2] = fmaf(xv[q + dx], wv.z, acc[q][2]);
                                acc[q][3] = fmaf(xv[q + dx], wv.w, acc[q][3]);
                            }
                        }
                    }
                }
            }
        }

        // ---- this region's contribution: gx += s_c * G_c ; gs[c] += sum_q x * G_c
        float4 sv = make_float4(0.f, 0.f, 0.f, 0.f);
        if (ci_ok) sv = __ldg(reinterpret_cast<const float4*>(p.s + ((int64_t)b * p.ncls + cls) * p.cin + ci));
        float ps[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            gxacc[q][0] = fmaf(sv.x, acc[q][0], gxacc[q][0]);
            gxacc[q][1] = fmaf(sv.y, acc[q][1], gxacc[q][1]);
            gxacc[q][2] = fmaf(sv.z, acc[q][2], gxacc[q][2]);
            gxacc[q][3] = fmaf(sv.w, acc[q][3], gxacc[q][3]);
            if (p.gs && p.x && valid[q] && ci_ok) {
                float4 xv = *reinterpret_cast<const float4*>(p.x + (((int64_t)b * p.h + qy) * p.w + qx0 + q) * p.cin + ci);
                ps[0] = fmaf(xv.x, acc[q][0], ps[0]);
                ps[1] = fmaf(xv.y, acc[q][1], ps[1]);
                ps[2] = fmaf(xv.z, acc[q][2], ps[2]);
                ps[3] = fmaf(xv.w, acc[q][3], ps[3]);
            }
        }
        if (p.gs && p.x) {
            __syncthreads();
            *reinterpret_cast<float4*>(red + pg * ICT + 4 * ig) = make_float4(ps[0], ps[1], ps[2], ps[3]);
            __syncthreads();
            if (threadIdx.x < ICT) {
                float t = 0.f;
                for (int g = 0; g < PG; ++g) t += red[g * ICT + threadIdx.x];
                if (i0 + threadIdx.x < p.cin) atomicAdd(p.gs + ((int64_t)b * p.ncls + cls) * p.cin + i0 + threadIdx.x, t);
            }
        }
    }

    if (p.gx && ci_ok) {
#pragma unroll
        for (int q = 0; q < 4; ++q)
            if (valid[q])
                *reinterpret_cast<float4*>(p.gx + (((int64_t)b * p.h + qy) * p.w + qx0 + q) * p.cin + ci) =
                    make_float4(gxacc[q][0], gxacc[q][1], gxacc[q][2], gxacc[q][3]);
    }
}

template <int ICG>
int launch_dgrad(const DgradParams& p0, cudaStream_t st) {
    DgradParams p = p0;
    constexpr int PG = 256 / ICG, TW = 4 * PG / TH, ICT = 4 * ICG;
    p.tiles_x = (int)e4s_ceil_div(p.w, TW);
    p.tiles_y = (int)e4s_ceil_div(p.h, TH);
    int64_t nblk = (int64_t)p.tiles_x * p.tiles_y * p.batch;
    if (nblk >= (1ll << 31)) return E4S_ERR_SHAPE;
    dim3 grid((unsigned)nblk, (unsigned)e4s_ceil_div(p.cin, ICT));
    size_t smem = sizeof(float) * (KC * (TH + 2) * (TW + 4) + KC * 9 * ICT + PG * ICT);
    static E4sSmemOptIn optin;
    if (const int rc = e4s_smem_optin(optin, modconv3x3_dgrad_kernel<ICG>, smem)) return rc;
    modconv3x3_dgrad_kernel<ICG><<<grid, 256, smem, st>>>(p);
    return e4s_launch_status();
}

// --------------------------------------------------------------------------------- class-segmented reduction
// gdu[b,c,o] += sum_{p in c} gv[p,o] * (v[p,o] - w_n n[p] - bias[o]),  gv = act'(y) gy,  v = act^-1(y)
// grid = (Cout/32 chunks, pixel splits, B); warp walks pixels, lane = channel.
constexpr int CR_WARPS = 8;
__global__ void __launch_bounds__(32 * CR_WARPS) class_reduce_kernel(const float* __restrict__ gy, const float* __restrict__ y,
                                                                     const uint8_t* __restrict__ label,
                                                                     const float* __restrict__ noise, const float* __restrict__ noise_w,
                                                                     const float* __restrict__ bias, float* __restrict__ gdu,
                                                                     int ncls, int hw, int cout, int noise_b, int act) {
    extern __shared__ float sums[];        // [CR_WARPS][ncls][32]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int b = blockIdx.z, o = blockIdx.x * 32 + lane;
    for (int i = threadIdx.x; i < CR_WARPS * ncls * 32; i += blockDim.x) sums[i] = 0.f;
    __syncthreads();
    const int per = (hw + gridDim.y - 1) / gridDim.y;
    const int p0 = blockIdx.y * per, p1 = min(hw, p0 + per);
    const float nw = (noise && noise_w) ? __ldg(noise_w) : 0.f;
    const float bo = (bias && o < cout) ? __ldg(bias + o) : 0.f;
    float* my = sums + warp * ncls * 32;
    for (int px = p0 + warp; px < p1; px += CR_WARPS) {
        if (o >= cout) break;
        const int cls = label ? min((int)label[(int64_t)b * hw + px], ncls - 1) : 0;
        const int64_t off = ((int64_t)b * hw + px) * cout + o;
        float g = gy[off], yv = y[off], v = yv;
        if (act) {
            g *= yv > 0.f ? SQRT2 : 0.2f * SQRT2;
            v = yv > 0.f ? yv * (1.0f / SQRT2) : yv * (1.0f / (0.2f * SQRT2));
        }
        float nz = noise ? nw * __ldg(noise + (int64_t)(noise_b == 1 ? 0 : b) * hw + px) : 0.f;
        my[cls * 32 + lane] += g * (v - nz - bo);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < ncls * 32; i += blockDim.x) {
        int cls = i >> 5, l = i & 31;
        float t = 0.f;
        for (int w = 0; w < CR_WARPS; ++w) t += sums[w * ncls * 32 + i];
        int oo = blockIdx.x * 32 + l;
        if (oo < cout && t != 0.f) atomicAdd(gdu + ((int64_t)b * ncls + cls) * cout + oo, t);
    }
}

// ------------------------------------------------------------------------------------------ ToRGB backward
// gx[p,i] = s[c(p),i] * t[p,i],  gs[b,c,i] += sum_{p in c} x[p,i] t[p,i],  t[p,i] = sum_o g[p,o] wrgb[o,i]
struct TorgbBwdParams {
    const float* g;        // planar [B, 3, H, W]
    const float* x;        // [B, H, W, Cin]
    const float* wrgb;     // [3, Cin]
    const float* s;        // [B, ncls, Cin]
    const uint8_t* label;
    float* gx;             // [B, H, W, Cin] or NULL
    float* gs;             // [B, ncls, Cin] or NULL (atomic accumulate)
    int batch, h, w, cin, ncls;
};

__global__ void __launch_bounds__(256) torgb_bwd_kernel(TorgbBwdParams p) {
    extern __shared__ __align__(16) float sm[];
    float* sw = sm;                          // [3][cin]
    float* ss = sw + 3 * p.cin;              // [ncls][cin]
    float* acc = ss + p.ncls * p.cin;        // [ncls][cin] style-gradient partials of this CTA
    const int b = blockIdx.y;
    for (int i = threadIdx.x; i < 3 * p.cin; i += 256) sw[i] = p.wrgb[i];
    for (int i = threadIdx.x; i < p.ncls * p.cin; i += 256) ss[i] = p.s[(int64_t)b * p.ncls * p.cin + i], acc[i] = 0.f;
    __syncthreads();
    const int64_t hw = (int64_t)p.h * p.w;
    const int nvec = p.cin / 4;
    // item = (pixel, 4-channel group); consecutive threads -> consecutive channel groups of one pixel
    const int64_t items = hw * nvec;
    for (int64_t it = (int64_t)blockIdx.x * 256 + threadIdx.x; it < items; it += (int64_t)gridDim.x * 256) {
        const int64_t pix = it / nvec;
        const int c = (int)(it - pix * nvec) * 4;
        const int cls = p.label ? min((int)p.label[(int64_t)b * hw + pix], p.ncls - 1) : 0;
        const float g0 = __ldg(p.g + ((int64_t)b * 3 + 0) * hw + pix), g1 = __ldg(p.g + ((int64_t)b * 3 + 1) * hw + pix),
                    g2 = __ldg(p.g + ((int64_t)b * 3 + 2) * hw + pix);
        float4 w0 = *reinterpret_cast<const float4*>(sw + c), w1 = *reinterpret_cast<const float4*>(sw + p.cin + c),
               w2 = *reinterpret_cast<const float4*>(sw + 2 * p.cin + c);
        float4 t;
        t.x = g0 * w0.x + g1 * w1.x + g2 * w2.x;
        t.y = g0 * w0.y + g1 * w1.y + g2 * w2.y;
        t.z = g0 * w0.z + g1 * w1.z + g2 * w2.z;
        t.w = g0 * w0.w + g1 * w1.w + g2 * w2.w;
        if (p.gx) {
            float4 sv = *reinterpret_cast<const float4*>(ss + cls * p.cin + c);
            st_stream_f4(p.gx + ((int64_t)b * hw + pix) * p.cin + c, make_float4(sv.x * t.x, sv.y * t.y, sv.z * t.z, sv.w * t.w));
        }
        if (p.gs) {
            float4 xv = ld_stream_f4(p.x + ((int64_t)b * hw + pix) * p.cin + c);
            float* a = acc + cls * p.cin + c;
            atomicAdd(a + 0, xv.x * t.x), atomicAdd(a + 1, xv.y * t.y), atomicAdd(a + 2, xv.z * t.z), atomicAdd(a + 3, xv.w * t.w);
        }
    }
    if (p.gs) {
        __syncthreads();
        for (int i = threadIdx.x; i < p.ncls * p.cin; i += 256)
            if (acc[i] != 0.f) atomicAdd(p.gs + (int64_t)b * p.ncls * p.cin + i, acc[i]);
    }
}

}  // namespace

extern "C" int e4s_modconv3x3_bwd_f32(const float* gy, const float* y, const float* x, const float* wd, const float* s,
                                      const float* demod, const uint8_t* label, float* gx, float* gs, int batch, int h,
                                      int w, int cin, int cout, int ncls, int up, int act, void* stream) {
    E4S_REQUIRE(gy && wd && s && (gx || gs), E4S_ERR_ARG);
    E4S_REQUIRE(!act || y, E4S_ERR_ARG);
    E4S_REQUIRE(!gs || x, E4S_ERR_ARG);
    E4S_REQUIRE(batch > 0 && h > 0 && w > 0 && cin > 0 && cout > 0 && ncls > 0, E4S_ERR_ARG);
    E4S_REQUIRE((cin % 4) == 0 && (cout % 4) == 0 && ncls <= MAXCLS, E4S_ERR_SHAPE);
    E4S_REQUIRE(label || ncls == 1, E4S_ERR_ARG);
    DgradParams p{gy, y, x, wd, s, demod, label, gx, gs, batch, h, w, cin, cout, ncls, up ? 1 : 0, act, 0, 0};
    cudaStream_t st = (cudaStream_t)stream;
    if (cin <= 32) return launch_dgrad<8>(p, st);
    return launch_dgrad<16>(p, st);
}

extern "C" int e4s_class_reduce_f32(const float* gy, const float* y, const uint8_t* label, const float* noise,
                                    const float* noise_w, const float* bias, float* gdu, int batch, int ncls, int ho,
                                    int wo, int cout, int noise_b, int act, void* stream) {
    E4S_REQUIRE(gy && y && gdu && batch > 0 && ncls > 0 && ncls <= MAXCLS && ho > 0 && wo > 0 && cout > 0, E4S_ERR_ARG);
    E4S_REQUIRE(label || ncls == 1, E4S_ERR_ARG);
    const int hw = ho * wo;
    int chunks = (int)e4s_ceil_div(cout, 32);
    int64_t want = e4s_ceil_div((int64_t)E4S_NUM_SMS * 4, (int64_t)chunks * batch);
    int splits = (int)(want < 1 ? 1 : want);
    int max_splits = (int)e4s_ceil_div(hw, 64);
    if (splits > max_splits) splits = max_splits;
    dim3 grid(chunks, splits, batch);
    size_t smem = sizeof(float) * CR_WARPS * ncls * 32;
    class_reduce_kernel<<<grid, 32 * CR_WARPS, smem, (cudaStream_t)stream>>>(gy, y, label, noise, noise_w, bias, gdu, ncls, hw,
                                                                           cout, noise_b, act);
    return e4s_launch_status();
}

extern "C" int e4s_torgb_bwd_f32(const float* g, const float* x, const float* wrgb, const float* s, const uint8_t* label,
                                 float* gx, float* gs, int batch, int h, int w, int cin, int ncls, void* stream) {
    E4S_REQUIRE(g && wrgb && s && (gx || gs) && batch > 0 && h > 0 && w > 0 && cin > 0 && ncls > 0, E4S_ERR_ARG);
    E4S_REQUIRE(!gs || x, E4S_ERR_ARG);
    E4S_REQUIRE((cin % 4) == 0 && ncls <= MAXCLS, E4S_ERR_SHAPE);
    E4S_REQUIRE(label || ncls == 1, E4S_ERR_ARG);
    size_t smem = sizeof(float) * (size_t)(3 + 2 * ncls) * cin;
    E4S_REQUIRE(smem <= 200 * 1024, E4S_ERR_SHAPE);
    static E4sSmemOptIn optin;
    if (const int rc = e4s_smem_optin(optin, torgb_bwd_kernel, smem)) return rc;
    TorgbBwdParams p{g, x, wrgb, s, label, gx, gs, batch, h, w, cin, ncls};
    int64_t items = (int64_t)h * w * (cin / 4);
    int64_t want = e4s_ceil_div(items, 256 * 8);
    int64_t cap = e4s_ceil_div((int64_t)E4S_NUM_SMS * 4, batch);
    if (cap < 1) cap = 1;
    dim3 grid((unsigned)(want < cap ? (want < 1 ? 1 : want) : cap), batch);
    torgb_bwd_kernel<<<grid, 256, smem, (cudaStream_t)stream>>>(p);
    return e4s_launch_status();
}
