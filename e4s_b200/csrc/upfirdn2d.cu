// upfirdn2d for sm_90a: zero-stuff (up), pad/crop, true 2-D convolution with a small FIR, decimate (down).
//
// Replaces upfirdn2d_kernel<> of the reference (src/models/stylegan2/op/upfirdn2d_kernel.cu:52-137),
// which stages tiles through `volatile` shared memory with scalar loads and 16 MACs per pixel from
// shared-memory taps.  This op is HBM-bound (8 B of traffic per output element), so the kernel is
// organised around memory, not math:
//   * hot configuration (up = down = 1, 4x4 FIR: the Blur after every up-sampling conv and its
//     gradient): one CTA streams a 128x32 (or 32x128) output tile; the input tile (+3 halo) is
//     staged once through shared memory with fully coalesced loads, FIR taps live in registers,
//     every thread produces a 4x4 micro-tile from two conflict-free 128-bit shared loads per input
//     row and writes 128-bit streaming stores;
//   * up = 2 with the 4x4 FIR (Upsample of the RGB skip, model.py:34-53): polyphase 2x2 stencil, one 128-bit
//     store of 4 outputs per thread;
//   * everything else (down = 2, odd FIR sizes): a gather kernel with the read-only path; these carry < 1 % of
//     the op's bytes in the model (SURVEY.md section 8a).
#include "common.cuh"

namespace {

struct UpfirdnParams {
    int in_h, in_w, out_h, out_w;
    int kh, kw;
    int up_x, up_y, down_x, down_y;
    int pad_x0, pad_y0;
};

// ----------------------------------------------------------------------------- generic gather
__global__ void __launch_bounds__(256) upfirdn2d_gather_kernel(const float* __restrict__ x, float* __restrict__ y,
                                                               const float* __restrict__ fir, UpfirdnParams p,
                                                               int64_t total) {
    __shared__ float sk[64];
    if (threadIdx.x < p.kh * p.kw) sk[threadIdx.x] = fir[threadIdx.x];
    __syncthreads();
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (int64_t)gridDim.x * blockDim.x) {
        int ox = (int)(idx % p.out_w);
        int64_t t = idx / p.out_w;
        int oy = (int)(t % p.out_h);
        int64_t plane = t / p.out_h;
        const float* xp = x + plane * (int64_t)p.in_h * p.in_w;
        // position of tap (ky,kx) of the FLIPPED kernel on the zero-stuffed, padded grid
        int my0 = oy * p.down_y - p.pad_y0;
        int mx0 = ox * p.down_x - p.pad_x0;
        float acc = 0.f;
        for (int ky = 0; ky < p.kh; ++ky) {
            int my = my0 + ky;
            if (my < 0 || my % p.up_y != 0) continue;
            int iy = my / p.up_y;
            if (iy >= p.in_h) continue;
            for (int kx = 0; kx < p.kw; ++kx) {
                int mx = mx0 + kx;
                if (mx < 0 || mx % p.up_x != 0) continue;
                int ix = mx / p.up_x;
                if (ix >= p.in_w) continue;
                acc += __ldg(xp + (int64_t)iy * p.in_w + ix) * sk[(p.kh - 1 - ky) * p.kw + (p.kw - 1 - kx)];
            }
        }
        y[idx] = acc;
    }
}

// ----------------------------------------------------------- up = 2, down = 1, 4x4 FIR (Upsample of the RGB skip)
// Polyphase form: on the zero-stuffed grid only taps of one parity per axis meet a sample, so an output is a 2x2
// stencil of the input, not 16 guarded taps.  One thread produces 4 consecutive output columns of one row (one
// 128-bit streaming store) from a 2 x 4 input window; the window is re-used by the neighbouring rows/threads
// through L1, so HBM sees each input once and the kernel is bound by its output stream (4x the input bytes).
__global__ void __launch_bounds__(256) upfirdn2d_up2_kernel(const float* __restrict__ x, float* __restrict__ y,
                                                            const float* __restrict__ fir, UpfirdnParams p,
                                                            int64_t total4) {
    float kf[4][4];                       // flipped taps: kf[ky][kx] multiplies the sample under tap (ky, kx)
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) kf[a][b] = __ldg(fir + (3 - a) * 4 + (3 - b));
    const int ow4 = p.out_w >> 2;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total4;
         idx += (int64_t)gridDim.x * blockDim.x) {
        const int q = (int)(idx % ow4);
        int64_t t = idx / ow4;
        const int oy = (int)(t % p.out_h);
        const int64_t plane = t / p.out_h;
        const float* xp = x + plane * (int64_t)p.in_h * p.in_w;
        // rows: taps ky = py, py + 2 land on even positions my = oy - pad_y0 + ky of the zero-stuffed grid
        const int my0 = oy - p.pad_y0, py = my0 & 1;
        const int iy0 = (my0 + py) >> 1;                       // sample under tap py; tap py + 2 sees iy0 + 1
        // columns: output ox = 4q + j, mx0 = ox - pad_x0; taps kx = px, px + 2; samples ix0(j), ix0(j) + 1
        const int base = 4 * q - p.pad_x0;
        const int c0 = (base + (base & 1)) >> 1;               // ceil(base / 2): leftmost sample any of the 4 outputs reads
        float v[2][4];
#pragma unroll
        for (int a = 0; a < 2; ++a) {
            const int iy = iy0 + a;
            const bool rowok = iy >= 0 && iy < p.in_h;
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                const int ix = c0 + c;
                v[a][c] = (rowok && ix >= 0 && ix < p.in_w) ? __ldg(xp + (int64_t)iy * p.in_w + ix) : 0.f;
            }
        }
        float o[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int mx0 = base + j, px = mx0 & 1;
            const int cj = ((mx0 + px) >> 1) - c0;             // 0..2
            float acc = 0.f;
#pragma unroll
            for (int a = 0; a < 2; ++a) {
                const float k0 = py ? (px ? kf[2 * a + 1][1] : kf[2 * a + 1][0]) : (px ? kf[2 * a][1] : kf[2 * a][0]);
                const float k1 = py ? (px ? kf[2 * a + 1][3] : kf[2 * a + 1][2]) : (px ? kf[2 * a][3] : kf[2 * a][2]);
                const float s0 = cj == 0 ? v[a][0] : (cj == 1 ? v[a][1] : v[a][2]);
                const float s1 = cj == 0 ? v[a][1] : (cj == 1 ? v[a][2] : v[a][3]);
                acc = fmaf(s0, k0, acc);
                acc = fmaf(s1, k1, acc);
            }
            o[j] = acc;
        }
        st_stream_f4(y + (plane * p.out_h + oy) * (int64_t)p.out_w + 4 * q, make_float4(o[0], o[1], o[2], o[3]));
    }
}

// ------------------------------------------------------------------- hot path: up=down=1, 4x4 FIR
// TXN x-threads per tile row, each owning 4 consecutive output columns; 256/TXN y-threads each owning
// 4 consecutive output rows.
template <int TXN>
__global__ void __launch_bounds__(256) upfirdn2d_fir4_kernel(const float* __restrict__ x, float* __restrict__ y,
                                                             const float* __restrict__ fir, UpfirdnParams p,
                                                             int tiles_x, int tiles_y) {
    constexpr int TYN = 256 / TXN;
    constexpr int TW = 4 * TXN, TH = 4 * TYN;
    constexpr int SW = TW + 4;      // staged columns (TW + 3 needed, rounded to a multiple of 4)
    constexpr int SH = TH + 3;
    __shared__ __align__(16) float tile[SH * SW];

    int bid = blockIdx.x;
    int tile_x = bid % tiles_x;
    bid /= tiles_x;
    int tile_y = bid % tiles_y;
    int64_t plane = bid / tiles_y;

    const int oy0 = tile_y * TH, ox0 = tile_x * TW;
    const int iy0 = oy0 - p.pad_y0, ix0 = ox0 - p.pad_x0;
    const float* xp = x + plane * (int64_t)p.in_h * p.in_w;

    // FIR taps in registers, flipped (true convolution, reference kernel.cu:77).
    float kf[4][4];
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) kf[a][b] = __ldg(fir + (3 - a) * 4 + (3 - b));

    // Stage the input tile, one warp per tile row: lane -> consecutive floats (coalesced), row/column validity is
    // a handful of compares per row instead of a div/mod per element.  All loads of a thread are issued before its
    // first shared store, so ~20-30 requests per thread are in flight.
    {
        constexpr int RPW = (SH + 7) / 8;            // rows per warp
        constexpr int CPL = (SW + 31) / 32;          // columns per lane
        const int wrp = threadIdx.x >> 5, ln = threadIdx.x & 31;
        float stage[RPW][CPL];
#pragma unroll
        for (int a = 0; a < RPW; ++a) {
            const int r = wrp + 8 * a;
            const int iy = iy0 + r;
            const bool rowok = (r < SH) && iy >= 0 && iy < p.in_h;
            const float* src = xp + (int64_t)iy * p.in_w + ix0;
#pragma unroll
            for (int c = 0; c < CPL; ++c) {
                const int col = ln + 32 * c, ix = ix0 + col;
                stage[a][c] = (rowok && col < SW && ix >= 0 && ix < p.in_w) ? ld_stream_f1(src + col) : 0.f;
            }
        }
#pragma unroll
        for (int a = 0; a < RPW; ++a) {
            const int r = wrp + 8 * a;
#pragma unroll
            for (int c = 0; c < CPL; ++c) {
                const int col = ln + 32 * c;
                if (r < SH && col < SW) tile[r * SW + col] = stage[a][c];
            }
        }
    }
    __syncthreads();

    const int tx = threadIdx.x % TXN, ty = threadIdx.x / TXN;
    float acc[4][4];
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) acc[a][b] = 0.f;

#pragma unroll
    for (int j = 0; j < 7; ++j) {
        const float4* rowp = reinterpret_cast<const float4*>(&tile[(4 * ty + j) * SW + 4 * tx]);
        float4 lo = rowp[0], hi = rowp[1];
        float v[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
#pragma unroll
        for (int orow = 0; orow < 4; ++orow) {
            int ky = j - orow;
            if (ky < 0 || ky > 3) continue;
#pragma unroll
            for (int oc = 0; oc < 4; ++oc)
#pragma unroll
                for (int kx = 0; kx < 4; ++kx) acc[orow][oc] = fmaf(v[oc + kx], kf[ky][kx], acc[orow][oc]);
        }
    }

    float* yp = y + plane * (int64_t)p.out_h * p.out_w;
    const int ox = ox0 + 4 * tx;
    const bool vec_ok = ((p.out_w & 3) == 0) && (ox + 3 < p.out_w);
#pragma unroll
    for (int orow = 0; orow < 4; ++orow) {
        int oy = oy0 + 4 * ty + orow;
        if (oy >= p.out_h) continue;
        float* dst = yp + (int64_t)oy * p.out_w + ox;
        if (vec_ok) {
            st_stream_f4(dst, make_float4(acc[orow][0], acc[orow][1], acc[orow][2], acc[orow][3]));
        } else {
#pragma unroll
            for (int oc = 0; oc < 4; ++oc)
                if (ox + oc < p.out_w) dst[oc] = acc[orow][oc];
        }
    }
}

}  // namespace

extern "C" int e4s_upfirdn2d_f32(const float* x, float* y, const float* fir, int planes, int in_h, int in_w,
                                 int out_h, int out_w, int kh, int kw, int up_x, int up_y, int down_x, int down_y,
                                 int pad_x0, int pad_x1, int pad_y0, int pad_y1, void* stream) {
    E4S_REQUIRE(x && y && fir, E4S_ERR_ARG);
    E4S_REQUIRE(planes > 0 && in_h > 0 && in_w > 0 && kh > 0 && kw > 0, E4S_ERR_ARG);
    E4S_REQUIRE(up_x > 0 && up_y > 0 && down_x > 0 && down_y > 0, E4S_ERR_ARG);
    E4S_REQUIRE(kh <= 8 && kw <= 8, E4S_ERR_SHAPE);
    // out size rule of the reference, upfirdn2d.py:100-101 / upfirdn2d_kernel.cu:167-168
    int eh = (in_h * up_y + pad_y0 + pad_y1 - kh) / down_y + 1;
    int ew = (in_w * up_x + pad_x0 + pad_x1 - kw) / down_x + 1;
    E4S_REQUIRE(eh == out_h && ew == out_w && out_h > 0 && out_w > 0, E4S_ERR_SHAPE);
    UpfirdnParams p{in_h, in_w, out_h, out_w, kh, kw, up_x, up_y, down_x, down_y, pad_x0, pad_y0};
    cudaStream_t st = (cudaStream_t)stream;
    const bool hot = (up_x == 1 && up_y == 1 && down_x == 1 && down_y == 1 && kh == 4 && kw == 4 &&
                      e4s_aligned16(y));
    if (hot) {
        if (out_w > 64) {
            int tx = (int)e4s_ceil_div(out_w, 128), ty = (int)e4s_ceil_div(out_h, 32);
            int64_t nblk = (int64_t)tx * ty * planes;
            E4S_REQUIRE(nblk < (1ll << 31), E4S_ERR_SHAPE);
            upfirdn2d_fir4_kernel<32><<<(unsigned)nblk, 256, 0, st>>>(x, y, fir, p, tx, ty);
        } else {
            int tx = (int)e4s_ceil_div(out_w, 32), ty = (int)e4s_ceil_div(out_h, 128);
            int64_t nblk = (int64_t)tx * ty * planes;
            E4S_REQUIRE(nblk < (1ll << 31), E4S_ERR_SHAPE);
            upfirdn2d_fir4_kernel<8><<<(unsigned)nblk, 256, 0, st>>>(x, y, fir, p, tx, ty);
        }
    } else if (up_x == 2 && up_y == 2 && down_x == 1 && down_y == 1 && kh == 4 && kw == 4 && (out_w & 3) == 0 &&
               e4s_aligned16(y)) {
        int64_t total4 = (int64_t)planes * out_h * (out_w >> 2);
        int64_t want = e4s_ceil_div(total4, 256), cap = (int64_t)E4S_NUM_SMS * 32;
        upfirdn2d_up2_kernel<<<(unsigned)(want < cap ? want : cap), 256, 0, st>>>(x, y, fir, p, total4);
    } else {
        int64_t total = (int64_t)planes * out_h * out_w;
        int64_t want = e4s_ceil_div(total, 256);
        int64_t cap = (int64_t)E4S_NUM_SMS * 32;  // grid-stride: a few waves of 8 CTAs/SM
        unsigned nblk = (unsigned)(want < cap ? want : cap);
        upfirdn2d_gather_kernel<<<nblk, 256, 0, st>>>(x, y, fir, p, total);
    }
    return e4s_launch_status();
}
