// Region-selected modulated 3x3 convolution, fp32 SIMT path (sm_90a).
//
// One launch = one StyledConv.forward of the reference (src/models/stylegan2/model.py:382-406) for ALL
// regions: where the reference runs the full modulated convolution once per region and mask-sums the
// twelve results (model.py:395-398), this kernel computes every output pixel exactly once with the
// style of that pixel's own region (bit-identical for one-hot masks, SURVEY.md App. A).  It uses the
// shared-weight form of the op (the reference's own non-fused branch, model.py:245-274):
//     y = demod[cls] * conv(x * s[cls], W / sqrt(9 Cin))
// so no per-sample weight tensor is ever materialised (the reference writes B*Cout*Cin*9 floats per
// region per layer, model.py:277-285).  Noise injection, bias and the sqrt(2)-scaled leaky ReLU
// (model.py:402-404) are fused into the epilogue: the activation makes one trip to HBM per layer.
//
// Up-sampling layers: conv_transpose2d(stride 2) followed by the [1,3,3,1] blur (model.py:287-300)
// is a polyphase filter: each of the four output parities is an ordinary 3x3 convolution over the
// INPUT grid with its own folded kernel (prepared once on the host side, DESIGN.md section 3).  The kernel
// treats the parity as one more tile coordinate.
//
// This is the exact-fp32 path: it serves the layers the tensor-core kernel does not take (4x4..16x16
// where tiles are mostly halo, odd shapes) and is the in-library cross-check for it.
//
// Tiling: CTA = 256 threads = OCG out-channel groups (4 channels each) x 256/OCG pixel groups
// (4 consecutive pixels of one row each); tile = 8 rows x TW columns x 4*OCG channels.  Cin is walked
// in chunks of 16 staged through shared memory: x tile with halo as [ci][row][col], weights as
// [ci][tap][co].  Inner loop per ci: 3 x (LDS.128 + LDS.64) for the x window, 9 x LDS.128 for the
// weights, 144 FMAs -> ~10 FMA per shared load, all shared accesses conflict-free or broadcast.
#include "common.cuh"

namespace {

constexpr int KC = 16;       // input channels per shared-memory chunk
constexpr int TH = 8;        // tile rows
constexpr int MAXCLS = 32;   // classes supported by the per-chunk style table

struct ModconvParams {
    const float* x;
    const float* wt;
    const float* s;
    const float* demod;
    const uint8_t* label;
    const float* noise;
    const float* noise_w;
    const float* bias;
    float* y;
    int batch, h, w, cin, cout, ncls, up, noise_b, act;
    int tiles_x, tiles_y;
};

template <int OCG>
__global__ void __launch_bounds__(256) modconv3x3_simt_kernel(ModconvParams p) {
    constexpr int PG = 256 / OCG;        // pixel groups
    constexpr int TW = 4 * PG / TH;      // tile columns (8 or 16)
    constexpr int XW = TW + 4;           // staged columns (TW + 2 used), multiple of 4
    constexpr int XR = TH + 2;
    constexpr int OCT = 4 * OCG;         // out channels per tile
    constexpr int XS_CI = XR * XW;       // floats per ci plane

    extern __shared__ __align__(16) float smem[];
    float* xs = smem;                          // [KC][XR][XW]
    float* ws = xs + KC * XS_CI;               // [KC][9][OCT]
    float* ss = ws + KC * 9 * OCT;             // [MAXCLS][KC]   (mixed tiles only)

    // ---- tile coordinates: blockIdx.x = ((b * nphase + phase) * tiles_y + ty) * tiles_x + tx
    int bid = blockIdx.x;
    const int tile_x = bid % p.tiles_x;
    bid /= p.tiles_x;
    const int tile_y = bid % p.tiles_y;
    bid /= p.tiles_y;
    const int nphase = p.up ? 4 : 1;
    const int phase = bid % nphase;
    const int b = bid / nphase;
    const int py = phase >> 1, px = phase & 1;
    const int co0 = blockIdx.y * OCT;

    const int og = threadIdx.x % OCG, pg = threadIdx.x / OCG;
    const int prow = pg / (TW / 4), pcol = 4 * (pg % (TW / 4));
    const int iy = tile_y * TH + prow;             // input-grid row of this thread's pixels
    const int ix0 = tile_x * TW + pcol;            // first of its 4 input-grid columns
    const int mul = p.up ? 2 : 1;
    const int ho = p.h * mul, wo = p.w * mul;
    const int oy = iy * mul + py;

    // ---- classes of this thread's output pixels; is the whole tile one class?
    int cls[4];
    bool valid[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        valid[q] = (iy < p.h) && (ix0 + q < p.w);
        cls[q] = 0;
        if (valid[q] && p.label) cls[q] = p.label[((int64_t)b * ho + oy) * wo + (ix0 + q) * mul + px];
        if (cls[q] >= p.ncls) cls[q] = p.ncls - 1;   // defensive: never index outside the style table
    }
    int tile_cls = 0;
    if (p.label) {
        // first pixel of the tile is always valid (tiles start inside the image)
        tile_cls = p.label[((int64_t)b * ho + (tile_y * TH) * mul + py) * wo + (tile_x * TW) * mul + px];
        if (tile_cls >= p.ncls) tile_cls = p.ncls - 1;
    }
    bool same = true;
#pragma unroll
    for (int q = 0; q < 4; ++q) same = same && (!valid[q] || cls[q] == tile_cls);
    const bool uniform = __syncthreads_and(same ? 1 : 0) != 0;

    float acc[4][4];
#pragma unroll
    for (int q = 0; q < 4; ++q)
#pragma unroll
        for (int o = 0; o < 4; ++o) acc[q][o] = 0.f;

    const float* xb = p.x + (int64_t)b * p.h * p.w * p.cin;
    const float* wph = p.wt + (int64_t)phase * 9 * p.cin * p.cout;
    const float* sb = p.s + (int64_t)b * p.ncls * p.cin;
    const int y_in0 = tile_y * TH - 1, x_in0 = tile_x * TW - 1;

    for (int ci0 = 0; ci0 < p.cin; ci0 += KC) {
        __syncthreads();   // previous chunk fully consumed
        // ---- stage x: one float4 = 4 input channels of one staged pixel
        for (int e = threadIdx.x; e < XR * (TW + 2) * (KC / 4); e += 256) {
            int cq = e % (KC / 4);
            int pix = e / (KC / 4);
            int r = pix / (TW + 2), c = pix - r * (TW + 2);
            int gy = y_in0 + r, gx = x_in0 + c, ci = ci0 + 4 * cq;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (gy >= 0 && gy < p.h && gx >= 0 && gx < p.w && ci < p.cin) {
                v = *reinterpret_cast<const float4*>(xb + ((int64_t)gy * p.w + gx) * p.cin + ci);
                if (uniform) {   // fold the style of the tile's single class into the activation
                    float4 sv = *reinterpret_cast<const float4*>(sb + (int64_t)tile_cls * p.cin + ci);
                    v.x *= sv.x, v.y *= sv.y, v.z *= sv.z, v.w *= sv.w;
                }
            }
            float* d = xs + (4 * cq) * XS_CI + r * XW + c;
            d[0] = v.x, d[XS_CI] = v.y, d[2 * XS_CI] = v.z, d[3 * XS_CI] = v.w;
        }
        // ---- stage weights: [ci][tap][co], float4 over co
        for (int e = threadIdx.x; e < KC * 9 * OCG; e += 256) {
            int c4 = e % OCG;
            int t = e / OCG;
            int tap = t % 9, ci = t / 9;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            int co = co0 + 4 * c4;
            if (ci0 + ci < p.cin && co < p.cout)
                v = __ldg(reinterpret_cast<const float4*>(wph + ((int64_t)tap * p.cin + ci0 + ci) * p.cout + co));
            *reinterpret_cast<float4*>(ws + (ci * 9 + tap) * OCT + 4 * c4) = v;
        }
        if (!uniform) {
            for (int e = threadIdx.x; e < p.ncls * KC; e += 256) {
                int c = e / KC, ci = e % KC;
                ss[e] = (ci0 + ci < p.cin) ? sb[(int64_t)c * p.cin + ci0 + ci] : 0.f;
            }
        }
        __syncthreads();

        if (uniform) {
#pragma unroll 4
            for (int ci = 0; ci < KC; ++ci) {
#pragma unroll
                for (int dy = 0; dy < 3; ++dy) {
                    const float* xr = xs + ci * XS_CI + (prow + dy) * XW + pcol;
                    float4 a = *reinterpret_cast<const float4*>(xr);
                    float2 c2 = *reinterpret_cast<const float2*>(xr + 4);
                    float xv[6] = {a.x, a.y, a.z, a.w, c2.x, c2.y};
#pragma unroll
                    for (int dx = 0; dx < 3; ++dx) {
                        float4 wv = *reinterpret_cast<const float4*>(ws + (ci * 9 + dy * 3 + dx) * OCT + 4 * og);
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
        } else {
            // mixed tile: the style factor depends on the OUTPUT pixel's class, so accumulate the
            // 9 taps of one input channel unscaled, then scale by that pixel's own s[cls][ci].
#pragma unroll 2
            for (int ci = 0; ci < KC; ++ci) {
                float tmp[4][4];
#pragma unroll
                for (int q = 0; q < 4; ++q)
#pragma unroll
                    for (int o = 0; o < 4; ++o) tmp[q][o] = 0.f;
#pragma unroll
                for (int dy = 0; dy < 3; ++dy) {
                    const float* xr = xs + ci * XS_CI + (prow + dy) * XW + pcol;
                    float4 a = *reinterpret_cast<const float4*>(xr);
                    float2 c2 = *reinterpret_cast<const float2*>(xr + 4);
                    float xv[6] = {a.x, a.y, a.z, a.w, c2.x, c2.y};
#pragma unroll
                    for (int dx = 0; dx < 3; ++dx) {
                        float4 wv = *reinterpret_cast<const float4*>(ws + (ci * 9 + dy * 3 + dx) * OCT + 4 * og);
#pragma unroll
                        for (int q = 0; q < 4; ++q) {
                            tmp[q][0] = fmaf(xv[q + dx], wv.x, tmp[q][0]);
                            tmp[q][1] = fmaf(xv[q + dx], wv.y, tmp[q][1]);
                            tmp[q][2] = fmaf(xv[q + dx], wv.z, tmp[q][2]);
                            tmp[q][3] = fmaf(xv[q + dx], wv.w, tmp[q][3]);
                        }
                    }
                }
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    float sv = ss[cls[q] * KC + ci];
#pragma unroll
                    for (int o = 0; o < 4; ++o) acc[q][o] = fmaf(sv, tmp[q][o], acc[q][o]);
                }
            }
        }
    }

    // ---- epilogue: demodulate, noise, bias, activation; 128-bit store of 4 channels
    const int co = co0 + 4 * og;
    if (co >= p.cout) return;
    const float nw = (p.noise && p.noise_w) ? __ldg(p.noise_w) : 0.f;
    float4 bv = make_float4(0.f, 0.f, 0.f, 0.f);
    if (p.bias) bv = __ldg(reinterpret_cast<const float4*>(p.bias + co));
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        if (!valid[q]) continue;
        const int ox = (ix0 + q) * mul + px;
        float4 d = make_float4(1.f, 1.f, 1.f, 1.f);
        if (p.demod) d = __ldg(reinterpret_cast<const float4*>(p.demod + ((int64_t)b * p.ncls + cls[q]) * p.cout + co));
        float nz = 0.f;
        if (p.noise) nz = nw * __ldg(p.noise + ((int64_t)(p.noise_b == 1 ? 0 : b) * ho + oy) * wo + ox);
        float4 r;
        r.x = acc[q][0] * d.x + nz + bv.x;
        r.y = acc[q][1] * d.y + nz + bv.y;
        r.z = acc[q][2] * d.z + nz + bv.z;
        r.w = acc[q][3] * d.w + nz + bv.w;
        if (p.act) {
            const float k = 1.41421356237309515f;
            r.x = lrelu_scaled(r.x, 0.2f, k), r.y = lrelu_scaled(r.y, 0.2f, k);
            r.z = lrelu_scaled(r.z, 0.2f, k), r.w = lrelu_scaled(r.w, 0.2f, k);
        }
        *reinterpret_cast<float4*>(p.y + (((int64_t)b * ho + oy) * wo + ox) * p.cout + co) = r;
    }
}

template <int OCG>
int launch_modconv(const ModconvParams& p0, cudaStream_t st) {
    ModconvParams p = p0;
    constexpr int PG = 256 / OCG, TW = 4 * PG / TH, OCT = 4 * OCG;
    p.tiles_x = (int)e4s_ceil_div(p.w, TW);
    p.tiles_y = (int)e4s_ceil_div(p.h, TH);
    int64_t nblk = (int64_t)p.tiles_x * p.tiles_y * (p.up ? 4 : 1) * p.batch;
    if (nblk >= (1ll << 31)) return E4S_ERR_SHAPE;
    dim3 grid((unsigned)nblk, (unsigned)e4s_ceil_div(p.cout, OCT));
    size_t smem = sizeof(float) * (KC * (TH + 2) * (TW + 4) + KC * 9 * OCT + MAXCLS * KC);
    static E4sSmemOptIn optin;
    if (const int rc = e4s_smem_optin(optin, modconv3x3_simt_kernel<OCG>, smem)) return rc;
    modconv3x3_simt_kernel<OCG><<<grid, 256, smem, st>>>(p);
    return e4s_launch_status();
}

// demod[r,o] = rsqrt(sum_i s[r,i]^2 wsq[o,i] + eps): one warp per (row, out channel)
__global__ void __launch_bounds__(256) demod_kernel(const float* __restrict__ s, const float* __restrict__ wsq,
                                                    float* __restrict__ demod, int rows, int cin, int cout, float eps) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= rows * cout) return;
    const int r = warp / cout, o = warp - r * cout;
    const float* sr = s + (int64_t)r * cin;
    const float* wr = wsq + (int64_t)o * cin;
    float acc = 0.f;
    for (int i = lane; i < cin; i += 32) {
        float v = sr[i];
        acc = fmaf(v * v, __ldg(wr + i), acc);
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
    if (lane == 0) demod[warp] = rsqrtf(acc + eps);
}

}  // namespace

extern "C" int e4s_demod_f32(const float* s, const float* wsq, float* demod, int rows, int cin, int cout, float eps,
                             void* stream) {
    E4S_REQUIRE(s && wsq && demod && rows > 0 && cin > 0 && cout > 0, E4S_ERR_ARG);
    int64_t warps = (int64_t)rows * cout;
    demod_kernel<<<(unsigned)e4s_ceil_div(warps * 32, 256), 256, 0, (cudaStream_t)stream>>>(s, wsq, demod, rows, cin, cout,
                                                                                            eps);
    return e4s_launch_status();
}

extern "C" int e4s_modconv3x3_fwd_f32(const float* x, const float* wt, const float* s, const float* demod,
                                      const uint8_t* label, const float* noise, const float* noise_w,
                                      const float* bias, float* y, int batch, int h, int w, int cin, int cout, int ncls,
                                      int up, int noise_b, int act, void* stream) {
    E4S_REQUIRE(x && wt && s && y, E4S_ERR_ARG);
    E4S_REQUIRE(batch > 0 && h > 0 && w > 0 && cin > 0 && cout > 0 && ncls > 0, E4S_ERR_ARG);
    E4S_REQUIRE((cin % 4) == 0 && (cout % 4) == 0 && ncls <= MAXCLS, E4S_ERR_SHAPE);
    E4S_REQUIRE(label || ncls == 1, E4S_ERR_ARG);
    E4S_REQUIRE(!noise || (noise_w && (noise_b == 1 || noise_b == batch)), E4S_ERR_ARG);
    E4S_REQUIRE(e4s_aligned16(x) && e4s_aligned16(wt) && e4s_aligned16(s) && e4s_aligned16(y) &&
                    (!demod || e4s_aligned16(demod)) && (!bias || e4s_aligned16(bias)),
                E4S_ERR_ALIGN);
    ModconvParams p{x, wt, s, demod, label, noise, noise_w, bias, y, batch, h, w, cin, cout, ncls, up ? 1 : 0,
                    noise_b, act, 0, 0};
    cudaStream_t st = (cudaStream_t)stream;
    if (cout <= 32) return launch_modconv<8>(p, st);
    return launch_modconv<16>(p, st);
}
