// conv3x3_rs_kernel: the forward 3x3 convolution on register operands - the plain modulated layers (any mask) and the
// plain convolutions of ESRGAN, ParseNet, RetinaFace, BiSeNet and face-vid2vid (plain, reflect-padded, 1x1, SPADE and
// volumetric modes) - and conv7x7_slices_kernel.
// conv3x3_wgmma_kernel (wgmma_conv_smem.cu) stages every operand element in shared memory as bf16 hi / lo planes and the MMAs read both operands
// from there: per K step ~112 KB cross the L1 / shared-memory data path for ~384 clocks of MMA.  Here shared memory holds
// the UNSCALED fp32 source pixels of a tile plus its 1-pixel halo (10 x 18 pixels x 32 channels, loaded once per channel
// chunk and read by all taps) and the weight tiles of every tap of the chunk, both copied by cp.async with no register
// round trip.  Each consumer thread builds its own rows of the wgmma A operand in registers: it reads the fp32 values
// at (row pixel + tap offset), multiplies them by the style of the row's own output pixel (held in registers for the
// chunk: the region does not change across taps) and splits them into bf16 hi / lo.  Only B is read from shared memory
// by the MMAs.
//
// A CTA is persistent and walks the work items blockIdx.x, + gridDim.x, ...; K runs chunk-outer, tap-inner.  A two-slot
// cp.async ring runs over the flattened (item, chunk) sequence, so the next tile's halo and weights arrive while the
// current chunk's MMAs run; one barrier per chunk.  The A fragments are double-buffered across taps: fragment set
// u = tap % 2 is rebuilt only after wgmma.wait_group has retired the MMAs of tap - 2 that read it.
// Resident weights: when the N tile's whole weight block (every chunk, every tap) fits in shared memory
// beside the two ring slots, it is copied once and stays; a slot then holds only the halo (and, at N = 32, the chunk's
// styles).  The N tile is the outermost index of an item, so a CTA reloads the block at most n_tiles - 1 times, after
// every MMA of the previous N tile has retired.  The MMAs read the same bytes in the same order either way: the results
// are bitwise identical.
// N = 128 (plain modulated layers with Cout % 128 == 0, nine taps, never resident): a chunk's weights (9 x 16 KB) do not
// fit twice.  The two slots hold only halos, and the weights stream through a ring of three slots of three taps each
// (after the halo slots, where the resident block would be) over the flattened (item, chunk, tap group) sequence: the
// next group's weights arrive while the current group's MMAs run, one barrier per group; the next chunk's halo and styles
// travel with its first group.  The slot invariant is written at the loop.  The sum order is the same as at N = 64
// (three products per K16 slice), so the results are bitwise identical to that width.
// The halo is an A tile (tile_at): pixel hp = (y + 1) * HALO_W + x + 1.
#include "wgmma_conv.cuh"

namespace wgmma_conv {

constexpr int HALO_H = TH + 2, HALO_W = TW + 2, HALO_PIX = HALO_H * HALO_W;
constexpr int HALO_BYTES = HALO_PIX * KC * 4;     // 23040

// FWD_DENSE, in the order of ESRGAN's modules: x5 = acc + bias; x5 * alpha + r0 (residual dense block); (...) * beta + r1
// (RRDB); leaky ReLU.  ro: offset of dst from p.out, where the residuals are read (each element by the thread storing it)
__device__ __forceinline__ void epilogue_dense2(const Params& p, int n, float a0, float a1, int64_t ro, float* dst) {
    float2 o = make_float2(a0, a1);
    if (p.bias) {
        const float2 bv = __ldg(reinterpret_cast<const float2*>(p.bias + n));
        o.x += bv.x, o.y += bv.y;
    }
    o.x *= p.alpha, o.y *= p.alpha;
    if (p.residual) {
        const float2 rv = *reinterpret_cast<const float2*>(p.residual + ro + n);
        o.x += rv.x, o.y += rv.y;
    }
    if (p.residual2) {
        const float2 rv = *reinterpret_cast<const float2*>(p.residual2 + ro + n);
        o.x = o.x * p.beta + rv.x, o.y = o.y * p.beta + rv.y;
    }
    if (p.lrelu != 1.f) {
        o.x = o.x > 0.f ? o.x : o.x * p.lrelu;
        o.y = o.y > 0.f ? o.y : o.y * p.lrelu;
    }
    *reinterpret_cast<float2*>(dst + n) = o;
}
// FWD_PW: t = (acc + bias) * alpha; t += r0; leaky ReLU; t += up (FPN's lateral + nearest-up-sampled coarser level), in
// that order; FACTOR (FWD_PWF): then t *= f.  ro as epilogue_dense2; up: the residual_up pixel of this output pixel, or NULL
template <bool FACTOR = false>
__device__ __forceinline__ void epilogue_pw2(const Params& p, int n, float a0, float a1, int64_t ro, const float* up, float f,
                                             float* dst) {
    float2 o = make_float2(a0, a1);
    if (p.bias) {
        const float2 bv = __ldg(reinterpret_cast<const float2*>(p.bias + n));
        o.x += bv.x, o.y += bv.y;
    }
    o.x *= p.alpha, o.y *= p.alpha;
    if (p.residual) {
        const float2 rv = *reinterpret_cast<const float2*>(p.residual + ro + n);
        o.x += rv.x, o.y += rv.y;
    }
    if (p.lrelu != 1.f) {
        o.x = o.x > 0.f ? o.x : o.x * p.lrelu;
        o.y = o.y > 0.f ? o.y : o.y * p.lrelu;
    }
    if (up) {
        const float2 uv = *reinterpret_cast<const float2*>(up + n);
        o.x += uv.x, o.y += uv.y;
    }
    if constexpr (FACTOR) o.x *= f, o.y *= f;
    *reinterpret_cast<float2*>(dst + n) = o;
}
// FWD_SPADE: columns n, n + 1 are (gamma, beta) of channel c = n / 2; xn = x s + t (the instance norm of x, s and t per
// sample and channel), o = xn (1 + (gamma + b_gamma)) + (beta + b_beta), then leaky ReLU with slope lrelu (1: none).
// xp: the input pixel of x, dst: the output pixel
__device__ __forceinline__ void epilogue_spade(const Params& p, int b, int n, float a0, float a1, const float* xp, float* dst) {
    const int c = n >> 1;
    const int64_t sc = (int64_t)b * (p.nch >> 1) + c;
    const float2 bv = __ldg(reinterpret_cast<const float2*>(p.bias + n));
    const float xn = fmaf(__ldg(xp + c), __ldg(p.s + sc), __ldg(p.shift + sc));
    float o = xn * (1.f + (a0 + bv.x)) + (a1 + bv.y);
    if (p.lrelu != 1.f) o = o > 0.f ? o : o * p.lrelu;
    dst[c] = o;
}

// FWD_VOL: mosaic pixel (my, mx) of a work item in pixel-tile row ty -> its cell and the pixel (ly, lx) of the cell's
// slice; false in a gutter, off the mosaic or past the last cell (VolGrid)
__device__ __forceinline__ bool vol_cell(const Params& p, int ty, int my, int mx, int& cell, int& ly, int& lx) {
    const VolGrid& v = p.vol;
    int cy = ty * TH / p.h, cx = 0;                   // gutter 0: the tile's cell
    if (v.gutter) cy = my / (p.h + 1), cx = mx / (p.w + 1);
    ly = my - cy * (p.h + v.gutter), lx = mx - cx * (p.w + v.gutter);
    cell = cy * v.ncx + cx;
    return my >= 0 && mx >= 0 && ly >= 0 && ly < p.h && lx >= 0 && lx < p.w && cx < v.ncx && cell < v.cells;
}

// Work items: (pixel tile, sample, N tile) (decode_item).  p.out_stride == 1, no up-sampling, no shift: the plain
// modulated convolution (epilogue: per-region demodulation, noise, bias, activation).  RES: resident weights - a
// compile-time choice, so that the streaming instantiation carries none of the resident mode's code.  stage: bytes of one ring slot, [halo | tap 0 w_hi | w_lo |
// tap 1 ...] when the weights stream, [halo] when resident or at N = 128 (the weight block follows the two slots: (chunk kc, tap ti)
// at (kc * ntaps + ti) * B_TAP).  Resident at N = 32 the kernel is compiled for two CTAs per SM (<= 128 registers): the
// next chunk's styles (its 32 channels of every region of the item's sample) wait in the slot after the halo instead of
// in registers.  Index arithmetic is 32-bit (the host checks the item count; a sample's activations and the weight
// planes stay below 2^31 elements), and the next (item, chunk) is decoded once, when its copies are issued.
// DENSE (every mode but FWD_RS): the plain convolution of ESRGAN's networks - no styles, labels or regions (the A
// fragments are the unscaled source values), the input read and the output written with pixel pitches p.a_ld / p.out_ld
// (channel slices of wider buffers: a residual dense block keeps x, x1 .. x4 in one [B, H, W, 160] buffer and its convs
// read and write disjoint channel ranges of it), optionally nearest 2x up-sampling in the halo copy, and epilogue_dense2.
// REFL (FWD_REFL): the halo outside the grid is the reflection padding of p.reflect instead of zero - GPEN's
// ParseNet; the zero-fill instantiations carry none of its code.
// PW (FWD_PW, FWD_PWF): the 1x1 convolution.  There is no halo: the 128 rows of an item are its 128 output pixels,
// read at (in_stride y, in_stride x) of the input, so a stride-2 shortcut needs no space-to-depth pass.  The tap loop runs
// over the p.ntaps 32-channel K chunks of a ring slot instead (slot: ntaps tiles of 128 pixels x 32 channels, then their
// ntaps weight tiles; K chunk c of the layer is tile c % ntaps of step c / ntaps), so one copy and one barrier cover
// 2 ntaps K16 slices.  Weights [2][Cout][Cin]; epilogue_pw2.
// VOL (FWD_VOL): the 3x3x3 convolution of face-vid2vid's 3D blocks over [B, H, W, D, Cin] -> [B, H, W, D,
// Cout] (pixel pitches p.a_ld = D Cin, p.out_ld = D Cout; H, W = p.h, p.w, the output grid).  The pixel tiles cover the
// mosaic p.vol (VolGrid, p.mh x p.mw, p.batch = 1): the halo copy maps each mosaic pixel to (cell, y, x), the cell to
// (b, z), and reads K chunk kc at depth z + kc / (Cin / 32) - 1, zero in gutters, past the last cell and outside the
// depth range; the store skips gutters.  Weights [2][9][Cout][3 Cin] (kz-major K); p.up is the (1, 2, 2) nearest
// up-sampling.  The zero-fill 2D instantiations carry none of its code.
// The choices above by MODE, for the kernel and its launcher: SPADE and FACTOR select epilogue_spade and epilogue_pw2's
// per-pixel factor
template <int MODE>
struct RsMode {
    static constexpr bool DENSE = MODE != FWD_RS, REFL = MODE == FWD_REFL, PW = MODE == FWD_PW || MODE == FWD_PWF,
                          VOL = MODE == FWD_VOL, SPADE = MODE == FWD_SPADE, FACTOR = MODE == FWD_PWF;
};
template <int NT, bool RES, int MODE>
__global__ void __launch_bounds__(NUM_THREADS, (NT == 32 && RES) ? 2 : 1)
    conv3x3_rs_kernel(const __grid_constant__ Params p, const int items, const int stage) {
    using R = RsMode<MODE>;
    static_assert(NT == 32 || NT == 64 || (NT == 128 && MODE == FWD_RS && !RES), "N tiles of 32 or 64, or streamed 128");
    constexpr int PW_TILE = M * KC * 4;                   // PW: one K chunk of the item's 128 pixels
    constexpr int B_PLANE = NT * KC * 2, B_TAP = 2 * B_PLANE;
    constexpr int B_CP = B_PLANE / 16;                    // 16-byte copies per (tap, plane)
    constexpr int B_PPI = B_CP < NUM_THREADS ? NUM_THREADS / B_CP : 1;    // (tap, plane) pairs per pass of the threads
    constexpr int TG = 3, W_SLOT = TG * B_TAP;            // N = 128: taps per weight-ring slot
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~uintptr_t(127));
    const uint32_t smem_s = (uint32_t)__cvta_generic_to_shared(smem);
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    // this thread's fragment rows: tile row `warp`, columns g and g + 8; fragment channels 8 j + 2 q, + 1 (j = 2 ks + half)
    const int g = lane >> 2, q = lane & 3;
    const int nchunks = p.kch / (R::PW ? KC * p.ntaps : KC), plane = p.nch * p.kch;
    const int H = p.h, W = p.w, MH = p.mh, MW = p.mw;
    // this thread's copies: channel quad t % 8 of halo pixels t / 8 + 32 i; weight row bn, quad bkq of the (tap, plane)
    // pairs bpl + B_PPI k
    const int hc = t & 7, bc = t % B_CP, bpl = t / B_CP;
    const int bn = (bc >> 5) * 8 + (bc & 7), bkq = (bc >> 3) & 3;
    const uint32_t b_dst = (bn >> 3) * SBO + bkq * LBO + (bn & 7) * 16;
    // where the next chunk's styles wait: in the ring slot (resident at N = 32) or in registers, loaded while the current
    // chunk's MMAs run
    constexpr bool STY_SMEM = NT == 32 && RES && !R::DENSE, STY_REG = !STY_SMEM && !R::DENSE;
    const int sty_ofs = R::PW ? p.ntaps * PW_TILE : HALO_BYTES, w_ofs = sty_ofs + (STY_SMEM ? p.ncls * KC * 4 : 0);    // in a ring slot
    const uint32_t w_s = smem_s + 2 * stage;              // resident weight block

    // region of each fragment row's own output pixel
    auto row_classes = [&](const Item& it, int (&c)[2]) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int iy = it.ty * TH + warp, ix = it.tx * TW + g + 8 * h;
            c[h] = (p.label && iy < MH && ix < MW) ? region(p.label, p.ncls, ((int64_t)it.b * MH + iy) * MW + ix) : 0;
        }
    };
    // this thread's styles of chunk kc (from ring slot `buf` when STY_SMEM): the fragment channels of each row's region
    auto load_styles = [&](const Item& it, int kc, int buf, const int (&c)[2], float2 (&sv)[2][4]) {
        const float* tab = STY_SMEM ? reinterpret_cast<const float*>(smem + buf * stage + sty_ofs)
                                    : p.s + (it.b * p.ncls) * p.kch + kc * KC;
        const int ld = STY_SMEM ? KC : p.kch;
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float2* v = reinterpret_cast<const float2*>(tab + c[h] * ld + 8 * j + 2 * q);
                sv[h][j] = STY_SMEM ? *v : __ldg(v);
            }
    };
    // weight tiles of chunk kc of the item's taps in the no-swizzle K-major core-matrix layout, tap ti at dst + ti * B_TAP
    auto copy_weights = [&](const Item& it, int kc, uint32_t dst) {
        const __nv_bfloat16* wb = p.wt + (it.n0 + bn) * p.kch + kc * KC + bkq * 8;
        for (int pl = bpl; pl < 2 * p.ntaps; pl += B_PPI) {
            const int ti = pl >> 1, hl = pl & 1;
            if constexpr (R::PW)
                cp_async16(dst + b_dst + ti * B_TAP + hl * B_PLANE, wb + hl * plane + (kc * (p.ntaps - 1) + ti) * KC, 16);
            else
                cp_async16(dst + b_dst + ti * B_TAP + hl * B_PLANE, wb + (hl * 9 + p.taps[ti]) * plane, 16);
        }
    };
    // the N tile's resident block: chunk kc's taps at w_s + kc * ntaps * B_TAP
    auto copy_block = [&](const Item& it) {
#pragma unroll 1
        for (int kc = 0; kc < nchunks; ++kc) copy_weights(it, kc, w_s + kc * p.ntaps * B_TAP);
    };
    // N = 128: weight-ring slot ws <- taps TG tg .. of chunk kc.  Copy c of a (tap, plane) is row 8 (c / 32) + c % 8,
    // channel quad (c / 8) % 4 of the tile: byte 16 c of the plane in the core-matrix layout
    auto copy_group = [&](const Item& it, int kc, int tg, int ws) {
        if constexpr (NT == 128) {
#pragma unroll
            for (int c = t; c < B_CP; c += NUM_THREADS) {
                const __nv_bfloat16* wb = p.wt + (it.n0 + (c >> 5) * 8 + (c & 7)) * p.kch + kc * KC + ((c >> 3) & 3) * 8;
#pragma unroll
                for (int pl = 0; pl < 2 * TG; ++pl)
                    cp_async16(w_s + ws * W_SLOT + pl * B_PLANE + c * 16, wb + ((pl & 1) * 9 + p.taps[TG * tg + (pl >> 1)]) * plane, 16);
            }
        }
    };
    // ring slot `buf` <- (item, chunk): the halo with zero fill outside the image (the convolution's padding) and the styles
    auto copy_halo = [&](const Item& it, int kc, int buf) {
        const uint32_t st = smem_s + buf * stage;
        if constexpr (R::PW) {
            // tile ti of the slot: K chunk kc * ntaps + ti of the item's pixels (pixel e = 16 row + column at e * 128 bytes,
            // an A tile); pixels off the output grid are zero-filled
            const float* xb = p.a + (int64_t)it.b * H * W * p.a_ld + kc * p.ntaps * KC + hc * 4;
            for (int e = t >> 3; e < p.ntaps * M; e += NUM_THREADS / 8) {
                const int ti = e / M, r = e % M, iy = it.ty * TH + (r >> 4), ix = it.tx * TW + (r & 15);
                const bool ok = iy < MH && ix < MW;
                const float* src = xb + (iy * p.in_stride * W + ix * p.in_stride) * p.a_ld + ti * KC;
                cp_async16(tile_at(st, e, hc), ok ? src : p.a, ok ? 16 : 0);
            }
            return;
        }
        const int sy0 = it.ty * TH - 1, sx0 = it.tx * TW - 1;
        if constexpr (R::VOL) {
            const int cin = p.kch / 3, nc = cin / KC, dz = kc / nc - 1, us = p.up, SH = H >> us, SW = W >> us;
            const float* xc = p.a + (kc - (dz + 1) * nc) * KC + hc * 4;
#pragma unroll
            for (int i = 0; i < (HALO_PIX * 8 + NUM_THREADS - 1) / NUM_THREADS; ++i) {
                const int hp = (t >> 3) + 32 * i;
                if (hp < HALO_PIX) {
                    const int hy = hp / HALO_W;
                    int cell, ly, lx;
                    bool ok = vol_cell(p, it.ty, sy0 + hy, sx0 + hp - hy * HALO_W, cell, ly, lx);
                    const int b = cell / p.vol.depth, z = cell - b * p.vol.depth + dz;
                    ok = ok && z >= 0 && z < p.vol.depth;
                    const float* src = xc + ((int64_t)(b * SH + (ly >> us)) * SW + (lx >> us)) * p.a_ld + z * p.vox_in;
                    cp_async16(tile_at(st, hp, hc), ok ? src : p.a, ok ? 16 : 0);
                }
            }
            return;
        }
        // DENSE with up-sampling: the source image is (H / 2) x (W / 2), pixel (sy, sx) of the grid reads (sy >> 1, sx >> 1)
        const int ld = R::DENSE ? p.a_ld : p.kch, us = R::DENSE ? p.up : 0, SW = W >> us;
        const float* xb = p.a + (int64_t)it.b * (H >> us) * SW * ld + kc * KC + hc * 4;
#pragma unroll
        for (int i = 0; i < (HALO_PIX * 8 + NUM_THREADS - 1) / NUM_THREADS; ++i) {
            const int hp = (t >> 3) + 32 * i;
            if (hp < HALO_PIX) {
                const int hy = hp / HALO_W, sy = sy0 + hy, sx = sx0 + hp - hy * HALO_W;
                if constexpr (R::REFL) {
                    // mirror (p.reflect == 1) or replicate, then clamp: pixels past a partial tile's edge stay in the
                    // image (they feed only outputs that are not stored)
                    int ry = sy, rx = sx;
                    if (p.reflect == 1) {
                        ry = sy < 0 ? -sy : (sy >= H ? 2 * H - 2 - sy : sy);
                        rx = sx < 0 ? -sx : (sx >= W ? 2 * W - 2 - sx : sx);
                    }
                    ry = min(max(ry, 0), H - 1), rx = min(max(rx, 0), W - 1);
                    cp_async16(tile_at(st, hp, hc), xb + ((ry >> us) * SW + (rx >> us)) * ld, 16);
                } else {
                    const bool ok = sy >= 0 && sy < H && sx >= 0 && sx < W;
                    cp_async16(tile_at(st, hp, hc), ok ? xb + ((sy >> us) * SW + (sx >> us)) * ld : p.a, ok ? 16 : 0);
                }
            }
        }
        if (STY_SMEM && t < p.ncls * (KC / 4))                        // ncls <= 32: one 16-byte copy per thread at most
            cp_async16(st + sty_ofs + t * 16, p.s + (it.b * p.ncls + (t >> 3)) * p.kch + kc * KC + (t & 7) * 4, 16);
    };
    // ... then, unless the weights are resident, the weight tiles of the item's taps (N = 128: of its first tap group,
    // into weight-ring slot ws)
    int ws = 0;
    auto prefetch = [&](const Item& it, int kc, int buf) {
        copy_halo(it, kc, buf);
        if constexpr (NT == 128)
            copy_group(it, kc, 0, ws);
        else if (!RES)
            copy_weights(it, kc, smem_s + buf * stage + w_ofs);
        cp_async_commit();
    };

    SplitAcc<NT> acc{};                               // zero: the fences read every register
    uint32_t fh[2][2][4], fl[2][2][4];                    // [tap % 2][K16 slice][register]: x_hi, x_lo fragments

    // a tap's fragments: this thread's rows g, g + 8 of tile row `warp` at the tap's offset (PW: of pixel tile `tap`)
    auto build = [&](const uint8_t* halo, int tap, const float2 (&sv)[2][4], uint32_t (&hi)[2][4], uint32_t (&lo)[2][4]) {
        const int dy = tap / 3, dx = tap % 3;
        auto hp = [&](int h) { return R::PW ? tap * M + warp * TW + g + 8 * h : (warp + dy) * HALO_W + g + 8 * h + dx; };
#pragma unroll
        for (int ks = 0; ks < 2; ++ks)
            build_frag(halo, hp, q, ks, hi[ks], lo[ks], R::DENSE ? nullptr : sv[0], R::DENSE ? nullptr : sv[1]);
    };

    // epilogue of an item: this thread's two rows of the tile, NT / 8 channel pairs each
    auto store_item = [&](const Item& it, const int (&c)[2]) {
        acc.fold();
        const float nw = (p.noise && p.noise_w) ? __ldg(p.noise_w) : 0.f;
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
            const int iy = it.ty * TH + warp, ix = it.tx * TW + g + 8 * hf;
            if (iy >= MH || ix >= MW) continue;
            if constexpr (R::VOL) {
                int cell, ly, lx;
                if (!vol_cell(p, it.ty, iy, ix, cell, ly, lx)) continue;
                const int b = cell / p.vol.depth, z = cell - b * p.vol.depth;
                const int64_t ro = (((int64_t)b * H + ly) * W + lx) * p.out_ld + z * p.vox_out;
#pragma unroll
                for (int nf = 0; nf < NT / 8; ++nf)
                    epilogue_dense2(p, it.n0 + nf * 8 + 2 * q, acc.d[4 * nf + 2 * hf], acc.d[4 * nf + 2 * hf + 1], ro, p.out + ro);
                continue;
            }
            if constexpr (R::DENSE) {
                const int64_t ro = (((int64_t)it.b * MH + iy) * MW + ix) * p.out_ld;
                if constexpr (R::SPADE) {
                    const int hs = p.norm_half;
                    const float* xp = p.norm_x + (((int64_t)it.b * (MH >> hs) + (iy >> hs)) * (MW >> hs) + (ix >> hs)) * p.norm_ld;
#pragma unroll
                    for (int nf = 0; nf < NT / 8; ++nf)
                        epilogue_spade(p, it.b, it.n0 + nf * 8 + 2 * q, acc.d[4 * nf + 2 * hf], acc.d[4 * nf + 2 * hf + 1], xp, p.out + ro);
                    continue;
                }
                if constexpr (R::PW) {
                    const float* up = p.residual_up ? p.residual_up + (((int64_t)it.b * (MH >> 1) + (iy >> 1)) * (MW >> 1) + (ix >> 1)) * p.rup_ld
                                                    : nullptr;
                    const float f = R::FACTOR ? __ldg(p.factor + ((int64_t)it.b * MH + iy) * MW + ix) : 1.f;
#pragma unroll
                    for (int nf = 0; nf < NT / 8; ++nf)
                        epilogue_pw2<R::FACTOR>(p, it.n0 + nf * 8 + 2 * q, acc.d[4 * nf + 2 * hf], acc.d[4 * nf + 2 * hf + 1], ro,
                                                        up, f, p.out + ro);
                    continue;
                }
#pragma unroll
                for (int nf = 0; nf < NT / 8; ++nf)
                    epilogue_dense2(p, it.n0 + nf * 8 + 2 * q, acc.d[4 * nf + 2 * hf], acc.d[4 * nf + 2 * hf + 1], ro, p.out + ro);
                continue;
            }
            const float z = p.noise ? nw * __ldg(p.noise + ((int64_t)(p.noise_b == 1 ? 0 : it.b) * MH + iy) * MW + ix) : 0.f;
            float* dst = p.out + (((int64_t)it.b * MH + iy) * MW + ix) * p.nch;
#pragma unroll
            for (int nf = 0; nf < NT / 8; ++nf) {
                const int n = it.n0 + nf * 8 + 2 * q;
                epilogue2<false>(p, it.b, c[hf], n, z, acc.d[4 * nf + 2 * hf], acc.d[4 * nf + 2 * hf + 1], dst);
            }
        }
    };

    int item = blockIdx.x;
    if (item >= items) return;
    Item cur = decode_item<false>(p, item, NT), nxt;
    int cls[2], cls_n[2];
    float2 sty[2][4], sty_n[2][4];                        // [row][j]: styles of the chunk's fragment channels
    row_classes(cur, cls);                               // DENSE: no label, every row region 0
    if (STY_REG) load_styles(cur, 0, 0, cls, sty);
    int kc = 0, buf = 0;
    // the next (item, chunk): decode it, start its copies into slot buf ^ 1 and load its styles
    auto fetch_next = [&](bool last_chunk, int item_n, int kc_n) {
        if (last_chunk) {
            nxt = decode_item<false>(p, item_n, NT);
            row_classes(nxt, cls_n);
        } else {
            nxt = cur, cls_n[0] = cls[0], cls_n[1] = cls[1];
        }
        prefetch(nxt, kc_n, buf ^ 1);
        if (STY_REG) load_styles(nxt, kc_n, 0, cls_n, sty_n);
    };
    if (RES) copy_block(cur);                            // committed with the first halo
    prefetch(cur, 0, 0);
#pragma unroll 1
    while (true) {
        const bool last_chunk = kc == nchunks - 1;
        const int item_n = last_chunk ? item + (int)gridDim.x : item, kc_n = last_chunk ? 0 : kc + 1;
        const bool more = item_n < items;
        if constexpr (NT == 128) {
            // The chunk's nine taps in TG-tap groups, one weight-ring slot each.  At a
            // group's barrier: its slot is complete and visible to the async proxy, and every thread has retired the MMAs
            // up to the first tap of the previous group (wait_group 1 before building that group's last tap; wait_group 0
            // at the end of a chunk) - so every MMA of the group before that, in both warpgroups.  Its slot, two groups
            // old, is the one refilled, once this group's first MMAs are issued; the previous group's slot may still be
            // read.  The halo slot refilled with the last group was last read by the builds of the previous chunk.
            const uint8_t* halo = smem + buf * stage;
#pragma unroll
            for (int tg = 0; tg < 9 / TG; ++tg) {
                cp_async_wait_all();
                fence_proxy_async();
                __syncthreads();
                const uint32_t bt0 = w_s + ws * W_SLOT;
                ws = ws == 2 ? 0 : ws + 1;                // the slot to refill
#pragma unroll
                for (int k = 0; k < TG; ++k) {
                    const int ti = TG * tg + k, u = ti & 1;
                    if (ti >= 2) wgmma_wait<1>();         // fragment set u: tap ti - 2, its last reader, has retired
                    build(halo, p.taps[ti], sty, fh[u], fl[u]);
                    issue_rs(acc, fh[u], fl[u], bt0 + k * B_TAP, kc == 0 && ti == 0);
                    if (k == 0) {
                        if (tg + 1 < 9 / TG) {
                            copy_group(cur, kc, tg + 1, ws);
                            cp_async_commit();
                        } else if (more) {
                            fetch_next(last_chunk, item_n, kc_n);
                        }
                    }
                }
            }
        } else {
            // slot buf complete and visible to the async proxy; every MMA of the previous chunk retired (wait_group 0 below),
            // so the other slot may be refilled once this chunk's first MMAs are issued
            cp_async_wait_all();
            fence_proxy_async();
            __syncthreads();
            const uint8_t* halo = smem + buf * stage;
            const uint32_t bt0 = RES ? w_s + kc * p.ntaps * B_TAP : smem_s + buf * stage + w_ofs;
            if (STY_SMEM) load_styles(cur, kc, buf, cls, sty);
            build(halo, p.taps[0], sty, fh[0], fl[0]);
            issue_rs(acc, fh[0], fl[0], bt0, kc == 0);
            if (more) fetch_next(last_chunk, item_n, kc_n);      // while the first tap's MMAs run
            // fragment set tap % 2 is rebuilt after wait_group 1 has retired tap - 2, its last reader
    #pragma unroll 1
            for (int ti = 1; ti < p.ntaps; ti += 2) {
                wgmma_wait<1>();
                build(halo, p.taps[ti], sty, fh[1], fl[1]);
                issue_rs(acc, fh[1], fl[1], bt0 + ti * B_TAP, false);
                if (ti + 1 < p.ntaps) {
                    wgmma_wait<1>();
                    build(halo, p.taps[ti + 1], sty, fh[0], fl[0]);
                    issue_rs(acc, fh[0], fl[0], bt0 + (ti + 1) * B_TAP, false);
                }
            }
        }
        wgmma_wait<0>();
        acc.fence();
        if (RES && more && nxt.n0 != cur.n0) {           // next N tile: its block, once both warpgroups' MMAs retired;
            __syncthreads();                              // the barrier at the top of the loop waits for the copies
            copy_block(nxt);
            cp_async_commit();
        }

        if (last_chunk) store_item(cur, cls);
        if (!more) break;
        cur = nxt, item = item_n, kc = kc_n, buf ^= 1;
        cls[0] = cls_n[0], cls[1] = cls_n[1];
        if (STY_REG) {
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int j = 0; j < 4; ++j) sty[h][j] = sty_n[h][j];
        }
    }
}

// ---- 7x7 convolution of every depth slice of a volume (face-vid2vid's dense-motion mask and occlusion, as one GEMM)
// x [B, H, W, D, Cin] -> y [B, D, H, W, 128]: y[b, z, y, x, n] = sum over (ky, kx, c) of w[ky 7 + kx, n, c] x[b, y + ky - 3,
// x + kx - 3, z, c], zero outside the slice; weights [2][49][128][Cin] (bf16 hi, lo).  One CTA per (8 x 16 pixel tile,
// slice): the A operand is built in registers from an fp32 halo tile (an A tile, tile_at, with a 3-pixel
// border: 14 x 22 pixels x 32 channels) and multiplied by the N = 128 weights of one tap with split_mma.  K runs
// chunk-outer, tap-inner: 49 taps of a 32-channel chunk, the chunk's halo loaded once.  The weights stream one tap per
// step through a ring of S7 slots (one cp.async group per step, PD7 = S7 - 2 steps ahead); the next chunk's halo travels
// with the first step of the current chunk, into the other halo slot.  The step invariant is written at the loop.  Every
// output's sum order is fixed by the channel count: bit reproducible and independent of the batch.
constexpr int K7_TAPS = 49, K7_R = 3, K7_HH = TH + 2 * K7_R, K7_HW = TW + 2 * K7_R, K7_HPIX = K7_HH * K7_HW;
constexpr int K7_HALO = K7_HPIX * KC * 4;               // 39424
constexpr int K7_NT = 128, K7_BPLANE = K7_NT * KC * 2, K7_BTAP = 2 * K7_BPLANE;
constexpr int S7 = 8, PD7 = S7 - 2;
constexpr size_t K7_SMEM = 128 + 2 * (size_t)K7_HALO + (size_t)S7 * K7_BTAP;

template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__global__ void __launch_bounds__(NUM_THREADS, 1)
    conv7x7_slices_kernel(const float* __restrict__ x, const __nv_bfloat16* __restrict__ wt, float* __restrict__ y, int depth,
                          int h, int w, int cin, int tiles_x) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~uintptr_t(127));
    const uint32_t smem_s = (uint32_t)__cvta_generic_to_shared(smem);
    const uint32_t w_s = smem_s + 2 * K7_HALO;
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5, g = lane >> 2, q = lane & 3, hc = t & 7;
    const int tx = blockIdx.x % tiles_x, ty = blockIdx.x / tiles_x, z = blockIdx.y, b = blockIdx.z;
    const int nsteps = (cin / KC) * K7_TAPS;
    const int64_t vp = (int64_t)depth * cin;              // pixel pitch of x

    // halo slot kc & 1 <- chunk kc of the tile's 14 x 22 pixels of slice z, zero outside the slice
    auto copy_halo = [&](int kc) {
        const uint32_t st = smem_s + (kc & 1) * K7_HALO;
        const float* xb = x + ((int64_t)b * h * w) * vp + (int64_t)z * cin + kc * KC + hc * 4;
        for (int hp = t >> 3; hp < K7_HPIX; hp += NUM_THREADS / 8) {
            const int hy = hp / K7_HW, sy = ty * TH - K7_R + hy, sx = tx * TW - K7_R + hp - hy * K7_HW;
            const bool ok = sy >= 0 && sy < h && sx >= 0 && sx < w;
            cp_async16(tile_at(st, hp, hc), ok ? xb + ((int64_t)sy * w + sx) * vp : x, ok ? 16 : 0);
        }
    };
    // weight slot s % S7 <- tap s % 49 of chunk s / 49, both planes in the no-swizzle K-major core-matrix layout (copy c
    // of a plane: row 8 (c / 32) + c % 8, channel quad (c / 8) % 4, at byte 16 c)
    auto copy_tap = [&](int s) {
        const int kc = s / K7_TAPS, tap = s - kc * K7_TAPS;
        const uint32_t dst = w_s + (s % S7) * K7_BTAP;
#pragma unroll
        for (int i = 0; i < 2 * K7_BPLANE / 16 / NUM_THREADS; ++i) {
            const int e = t + NUM_THREADS * i, hl = e / (K7_BPLANE / 16), c = e % (K7_BPLANE / 16);
            const int n = (c >> 5) * 8 + (c & 7);
            cp_async16(dst + hl * K7_BPLANE + c * 16,
                       wt + ((int64_t)(hl * K7_TAPS + tap) * K7_NT + n) * cin + kc * KC + ((c >> 3) & 3) * 8, 16);
        }
    };

    SplitAcc<K7_NT> acc{};                                // zero: the fences read every register
    uint32_t fh[2][2][4], fl[2][2][4];                    // [step % 2][K16 slice][register]: x_hi, x_lo fragments
    // a tap's fragments: this thread's rows g, g + 8 of tile row `warp` at the tap's offset
    auto build = [&](const uint8_t* halo, int tap, uint32_t (&hi)[2][4], uint32_t (&lo)[2][4]) {
        const int dy = tap / 7, dx = tap % 7;
        auto hp = [&](int h) { return (warp + dy) * K7_HW + g + 8 * h + dx; };
#pragma unroll
        for (int ks = 0; ks < 2; ++ks) build_frag(halo, hp, q, ks, hi[ks], lo[ks]);
    };

    copy_halo(0);
    for (int s = 0; s < PD7; ++s) {                       // one group per step: step 0 carries chunk 0's halo
        if (s < nsteps) copy_tap(s);
        cp_async_commit();
    }
#pragma unroll 1
    for (int s = 0; s < nsteps; ++s) {
        // Step s: groups 0 .. s + PD7 - 1 are committed, so waiting for all but the newest PD7 - 1 completes group s (its
        // weights and, at a chunk's first step, the halo issued one chunk earlier).  Past the barrier every thread has
        // retired the MMAs of step s - 2 (wait_group 1 after issuing step s - 1): its fragment set (s & 1) and weight
        // slot ((s + PD7) % S7) are free.  The other halo slot was last read by the builds of the previous chunk.
        cp_async_wait<PD7 - 1>();
        fence_proxy_async();
        __syncthreads();
        const int kc = s / K7_TAPS, tap = s - kc * K7_TAPS, u = s & 1;
        build(smem + (kc & 1) * K7_HALO, tap, fh[u], fl[u]);
        issue_rs(acc, fh[u], fl[u], w_s + (s % S7) * K7_BTAP, s == 0);
        if (tap == 0 && (kc + 1) * K7_TAPS < nsteps) copy_halo(kc + 1);
        if (s + PD7 < nsteps) copy_tap(s + PD7);
        cp_async_commit();
        wgmma_wait<1>();
    }
    wgmma_wait<0>();
    acc.fence();
    acc.fold();
    // this thread's rows g, g + 8 of tile row `warp`; register 4 nf + 2 hf + e: column 8 nf + 2 q + e
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) {
        const int iy = ty * TH + warp, ix = tx * TW + g + 8 * hf;
        float* dst = y + ((((int64_t)b * depth + z) * h + iy) * w + ix) * K7_NT + 2 * q;
#pragma unroll
        for (int nf = 0; nf < K7_NT / 8; ++nf)
            *reinterpret_cast<float2*>(dst + nf * 8) = make_float2(acc.d[4 * nf + 2 * hf], acc.d[4 * nf + 2 * hf + 1]);
    }
}

// ------------------------------------------------------------------------------------------ host
template <int NT, int MODE>
static int launch_rs(Params p, cudaStream_t st) {
    using R = RsMode<MODE>;
    p.n_tiles = p.nch / NT;
    const int64_t items = (int64_t)p.tiles_x * p.tiles_y * p.batch * p.n_tiles;
    // persistent, as many CTAs per SM as fit (the two ring slots of a 64-channel tile with nine streamed taps take
    // 189 KB of shared memory)
    const int64_t ld = R::DENSE ? (p.a_ld > p.out_ld ? p.a_ld : p.out_ld) : p.kch;
    if (items >= (1ll << 31) - 1024 || (int64_t)p.h * p.w * ld >= (1ll << 31) || 18ll * p.nch * p.kch >= (1ll << 31))
        return E4S_ERR_SHAPE;
    // the weights stay resident when the N tile's whole block fits beside the two ring slots (halo and styles);
    // E4S_B200_RS_STREAM=1 streams them with every chunk regardless (tests)
    // (PW: the "taps" are the K chunks of a slot, the block is every chunk once, the halo the slot's pixel tiles)
    const int64_t tap_bytes = 2 * NT * KC * 2, block = (int64_t)(p.kch / KC) * (R::PW ? 1 : p.ntaps) * tap_bytes;
    const int halo = R::PW ? p.ntaps * M * KC * 4 : HALO_BYTES;
    const int res_slot = halo + (NT == 32 && !R::DENSE ? p.ncls * KC * 4 : 0);   // resident ring slot: halo (, styles)
    const char* f = getenv("E4S_B200_RS_STREAM");
    // N = 128: never resident; the two slots hold halos, and a ring of three 3-tap weight slots follows them (190 KB)
    constexpr bool WIDE = NT == 128;
    if (WIDE && p.ntaps != 9) return E4S_ERR_SHAPE;
    const bool resident = !WIDE && !(f && atoi(f) != 0) && 128 + 2 * res_slot + block <= e4s_smem_optin_limit();
    const int stage = resident || WIDE ? res_slot : halo + p.ntaps * (int)tap_bytes;
    const size_t smem = 128 + 2 * (size_t)stage + (resident ? (size_t)block : WIDE ? 9 * (size_t)tap_bytes : 0);
    static E4sSmemOptIn optin[2];
    static E4sOccupancy occ[2];
    auto kernel = conv3x3_rs_kernel<NT, false, MODE>;
    if constexpr (!WIDE)
        if (resident) kernel = conv3x3_rs_kernel<NT, true, MODE>;
    if (const int rc = e4s_smem_optin(optin[resident], kernel, smem)) return rc;
    const int per_sm = e4s_ctas_per_sm(occ[resident], kernel, NUM_THREADS, smem);
    const int64_t slots = (int64_t)num_sms() * (per_sm > 1 ? per_sm : 1);
    const int64_t grid = items < slots ? items : slots;
    kernel<<<(unsigned)grid, NUM_THREADS, smem, st>>>(p, (int)items, stage);
    return e4s_launch_status();
}

// nt: channels per work item (pick_ntile, or 128 at FWD_RS: pick_ntile_rs)
template <int MODE>
static int launch(const Params& p, int nt, cudaStream_t st) {
    if (nt == 32) return launch_rs<32, MODE>(p, st);
    if constexpr (MODE == FWD_RS)
        if (nt == 128) return launch_rs<128, MODE>(p, st);
    return launch_rs<64, MODE>(p, st);
}

// N-tile width of the plain modulated layers on the register-operand kernel: 128 when the channel count allows it and
// the 64-channel items would not fit in one wave of CTAs (one per SM), else pick_ntile's choice.  A 128-channel item
// takes ~1.5x the time of a 64-channel one (0.186 against 0.124 ms at 512 -> 512 channels): 1.27 - 1.33x faster where
// both widths run several waves or 128 saves one of two, 0.67x where 64 already ran in one (H100 80GB HBM3, 700 W;
// DESIGN.md section 9).  E4S_B200_RS_NTILE=64|128 forces a width the channel count allows; a set E4S_B200_NTILE keeps
// pick_ntile's choice.
static int pick_ntile_rs(int channels, int64_t pixel_tiles) {
    const char* f = getenv("E4S_B200_RS_NTILE");
    const int v = f ? atoi(f) : 0;
    if ((v == 64 || v == 128) && channels % v == 0) return v;
    if (channels % 128 == 0 && !getenv("E4S_B200_NTILE") && 2 * pixel_tiles * (channels / 128) > num_sms()) return 128;
    return pick_ntile(channels, pixel_tiles);
}

// plain modulated convolution (p.up == 0, p.out_stride == 1, no shift): the register-operand kernel
static int forward_rs(Params p, cudaStream_t st) {
    tiles(p);
    const int nt = pick_ntile_rs(p.nch, (int64_t)p.tiles_x * p.tiles_y * p.batch);
    return launch<FWD_RS>(p, nt, st);
}

}  // namespace wgmma_conv

extern "C" int e4s_modconv3x3_tcr_fwd(const float* x, const void* w_hilo_bf16, const float* s, const float* demod,
                                      const uint8_t* label, const float* noise, const float* noise_w, const float* bias,
                                      float* y, int batch, int h, int w, int cin, int cout, int ncls, int up, int noise_b,
                                      int act, void* stream) {
    if (const int rc = wgmma_conv::check_modconv_fwd(x, w_hilo_bf16, s, demod, label, noise, noise_w, bias, y, batch, h, w,
                                                     cin, cout, ncls, noise_b, true))
        return rc;
    wgmma_conv::Params p{};
    p.a = x, p.wt = static_cast<const __nv_bfloat16*>(w_hilo_bf16), p.s = s, p.demod = demod, p.label = label;
    p.noise = noise, p.noise_w = noise_w, p.bias = bias, p.out = y;
    p.batch = batch, p.h = h, p.w = w, p.kch = cin, p.nch = cout, p.ncls = ncls, p.noise_b = noise_b, p.act = act ? 1 : 0;
    p.up = up ? 1 : 0;
    wgmma_conv::set_taps(p, 0);
    return up ? wgmma_conv::forward(p, (cudaStream_t)stream) : wgmma_conv::forward_rs(p, (cudaStream_t)stream);
}

// Host-only: the N-tile width forward_rs picks for this shape (see pick_ntile_rs); no launch, no device access beyond the
// SM count.
extern "C" int e4s_modconv3x3_tcr_fwd_plan(int batch, int h, int w, int cout, int* ntile) {
    E4S_REQUIRE(ntile && batch > 0 && h > 0 && w > 0 && cout > 0, E4S_ERR_ARG);
    E4S_REQUIRE((cout % 32) == 0, E4S_ERR_SHAPE);
    *ntile = wgmma_conv::pick_ntile_rs(cout, e4s_ceil_div(w, wgmma_conv::TW) * e4s_ceil_div(h, wgmma_conv::TH) * batch);
    return E4S_OK;
}

// The plain-mode entries' checks and parameters (p.reflect = reflect for FWD_REFL); up: the halo reads the input at
// (sy >> up, sx >> up) (nearest up-sampling by 2^up; h, w: the input grid)
static int dense_params(wgmma_conv::Params& p, const float* x, int x_ld, const void* w_hilo_bf16, const float* bias, float alpha,
                        const float* r0, float beta, const float* r1, float* y, int y_ld, int batch, int h, int w, int cin,
                        int cout, int up, int reflect, int tap_mask, float lrelu_slope) {
    E4S_REQUIRE(x && w_hilo_bf16 && y, E4S_ERR_ARG);
    E4S_REQUIRE(batch > 0 && h > 0 && w > 0 && cin > 0 && cout > 0 && x_ld >= cin && y_ld >= cout, E4S_ERR_ARG);
    E4S_REQUIRE(up >= 0 && up <= 2, E4S_ERR_ARG);
    E4S_REQUIRE((cin % 32) == 0 && (cout % 32) == 0, E4S_ERR_SHAPE);
    E4S_REQUIRE((x_ld % 4) == 0 && (y_ld % 4) == 0, E4S_ERR_ALIGN);
    E4S_REQUIRE(e4s_aligned16(x) && e4s_aligned16(w_hilo_bf16) && e4s_aligned16(y), E4S_ERR_ALIGN);
    for (const void* q : {(const void*)bias, (const void*)r0, (const void*)r1}) E4S_REQUIRE(!q || e4s_aligned16(q), E4S_ERR_ALIGN);
    const int m = 1 << up;
    p.a = x, p.wt = static_cast<const __nv_bfloat16*>(w_hilo_bf16), p.bias = bias, p.out = y;
    p.residual = r0, p.residual2 = r1, p.alpha = alpha, p.beta = beta, p.lrelu = lrelu_slope;
    p.a_ld = x_ld, p.out_ld = y_ld, p.up = up, p.reflect = reflect;
    p.batch = batch, p.h = h * m, p.w = w * m, p.kch = cin, p.nch = cout, p.ncls = 1;
    wgmma_conv::set_taps(p, tap_mask);
    wgmma_conv::tiles(p);
    return E4S_OK;
}

// The plain-mode entries: checks, then the launch of MODE (FWD_DENSE: zero padding; FWD_REFL: p.reflect = reflect) at N
// tile ntile (0: pick_ntile's choice for the launch size).
template <int MODE>
static int dense_conv(const float* x, int x_ld, const void* w_hilo_bf16, const float* bias, float alpha, const float* r0,
                      float beta, const float* r1, float* y, int y_ld, int batch, int h, int w, int cin, int cout, int up,
                      int reflect, int tap_mask, float lrelu_slope, void* stream, int ntile = 0) {
    wgmma_conv::Params p{};
    if (const int rc = dense_params(p, x, x_ld, w_hilo_bf16, bias, alpha, r0, beta, r1, y, y_ld, batch, h, w, cin, cout, up,
                                    reflect, tap_mask, lrelu_slope))
        return rc;
    const int nt = ntile ? ntile : wgmma_conv::pick_ntile(cout, (int64_t)p.tiles_x * p.tiles_y * batch);
    return wgmma_conv::launch<MODE>(p, nt, (cudaStream_t)stream);
}

extern "C" int e4s_conv3x3_dense_tcr_f32(const float* x, int x_ld, const void* w_hilo_bf16, const float* bias, float alpha,
                                         const float* r0, float beta, const float* r1, float* y, int y_ld, int batch, int h,
                                         int w, int cin, int cout, int up, float lrelu_slope, void* stream) {
    return dense_conv<wgmma_conv::FWD_DENSE>(x, x_ld, w_hilo_bf16, bias, alpha, r0, beta, r1, y, y_ld, batch, h, w, cin, cout,
                                             up ? 1 : 0, 0, 0, lrelu_slope, stream);
}

extern "C" int e4s_conv3x3_reflect_tcr_f32(const float* x, int x_ld, const void* w_hilo_bf16, const float* bias, float alpha,
                                           const float* r0, float beta, const float* r1, float* y, int y_ld, int batch, int h,
                                           int w, int cin, int cout, int mode, float lrelu_slope, void* stream) {
    E4S_REQUIRE(mode >= 0 && mode <= 2, E4S_ERR_ARG);
    E4S_REQUIRE(h >= 2 && w >= 2, E4S_ERR_SHAPE);
    // mode 0: stride 1, mirror; 1: nearest 2x up-sampling, replicate; 2: stride 2 over the space-to-depth operand (taps
    // {-1, 0}^2), replicate
    return dense_conv<wgmma_conv::FWD_REFL>(x, x_ld, w_hilo_bf16, bias, alpha, r0, beta, r1, y, y_ld, batch, h, w, cin, cout,
                                            mode == 1, mode == 0 ? 1 : 2, mode == 2 ? 0x1B : 0, lrelu_slope, stream);
}

extern "C" int e4s_conv3x3_zero_tcr_f32(const float* x, int x_ld, const void* w_hilo_bf16, const float* bias, float alpha,
                                        const float* r0, float beta, const float* r1, float* y, int y_ld, int batch, int h, int w,
                                        int cin, int cout, int stride, float lrelu_slope, void* stream) {
    E4S_REQUIRE(stride == 1 || stride == 2, E4S_ERR_ARG);
    // zero padding 1; stride 2 over the space-to-depth operand: the taps (dy, dx) in {-1, 0}^2.  The N tile follows the
    // channel count only, so each output's sum order (and value) does not depend on the batch
    return dense_conv<wgmma_conv::FWD_DENSE>(x, x_ld, w_hilo_bf16, bias, alpha, r0, beta, r1, y, y_ld, batch, h, w, cin, cout,
                                             0, 0, stride == 2 ? 0x1B : 0, lrelu_slope, stream, (cout % 64) == 0 ? 64 : 32);
}

extern "C" int e4s_conv3x3_zero_up_tcr_f32(const float* x, int x_ld, const void* w_hilo_bf16, const float* bias, float* y,
                                           int y_ld, int batch, int h, int w, int cin, int cout, int up_shift, float lrelu_slope,
                                           void* stream) {
    E4S_REQUIRE(up_shift == 1 || up_shift == 2, E4S_ERR_ARG);
    // e4s_conv3x3_zero_tcr_f32 over the nearest up-sampling of x by 2^up_shift, read through the halo copy (the
    // up-sampled input is never written); the N tile follows the channel count only
    return dense_conv<wgmma_conv::FWD_DENSE>(x, x_ld, w_hilo_bf16, bias, 1.f, nullptr, 1.f, nullptr, y, y_ld, batch, h, w, cin,
                                             cout, up_shift, 0, 0, lrelu_slope, stream, (cout % 64) == 0 ? 64 : 32);
}

extern "C" int e4s_spade_tcr_f32(const float* actv, int actv_ld, const void* w_hilo_bf16, const float* bias, const float* x,
                                 int x_ld, int x_half, const float* scale, const float* shift, float* y, int y_ld, int batch,
                                 int h, int w, int cin, int c, float lrelu_slope, void* stream) {
    E4S_REQUIRE(bias && x && scale && shift && x_ld >= c && y_ld >= c && (x_half == 0 || x_half == 1), E4S_ERR_ARG);
    E4S_REQUIRE(!x_half || ((h % 2) == 0 && (w % 2) == 0), E4S_ERR_SHAPE);
    wgmma_conv::Params p{};
    // the GEMM's 2 C columns are the (gamma, beta) pairs; its output pitch is unused (the epilogue stores C channels)
    if (const int rc = dense_params(p, actv, actv_ld, w_hilo_bf16, bias, 1.f, nullptr, 1.f, nullptr, y, 2 * c, batch, h, w, cin,
                                    2 * c, 0, 0, 0, lrelu_slope))
        return rc;
    p.out_ld = y_ld, p.norm_x = x, p.norm_ld = x_ld, p.norm_half = x_half, p.s = scale, p.shift = shift;
    // the N tile follows the channel count only: bit identical at any batch
    return wgmma_conv::launch<wgmma_conv::FWD_SPADE>(p, (2 * c) % 64 == 0 ? 64 : 32, (cudaStream_t)stream);
}

// The pointwise entries' checks and parameters
static int pw_params(wgmma_conv::Params& p, const float* x, int x_ld, const void* w_hilo_bf16, const float* bias, float alpha,
                     const float* r0, const float* r_up, int r_up_ld, float* y, int y_ld, int batch, int h, int w, int cin,
                     int cout, int stride, float lrelu_slope) {
    E4S_REQUIRE(x && w_hilo_bf16 && y, E4S_ERR_ARG);
    E4S_REQUIRE(batch > 0 && h > 0 && w > 0 && cin > 0 && cout > 0 && x_ld >= cin && y_ld >= cout, E4S_ERR_ARG);
    E4S_REQUIRE(stride == 1 || stride == 2, E4S_ERR_ARG);
    E4S_REQUIRE(!r_up || r_up_ld >= cout, E4S_ERR_ARG);
    E4S_REQUIRE((cin % 32) == 0 && (cout % 32) == 0 && (!r_up || ((h % 2) == 0 && (w % 2) == 0)), E4S_ERR_SHAPE);
    E4S_REQUIRE((x_ld % 4) == 0 && (y_ld % 4) == 0 && (!r_up || (r_up_ld % 4) == 0), E4S_ERR_ALIGN);
    E4S_REQUIRE(e4s_aligned16(x) && e4s_aligned16(w_hilo_bf16) && e4s_aligned16(y), E4S_ERR_ALIGN);
    for (const void* q : {(const void*)bias, (const void*)r0, (const void*)r_up}) E4S_REQUIRE(!q || e4s_aligned16(q), E4S_ERR_ALIGN);
    p.a = x, p.wt = static_cast<const __nv_bfloat16*>(w_hilo_bf16), p.bias = bias, p.out = y;
    p.residual = r0, p.residual_up = r_up, p.rup_ld = r_up_ld, p.alpha = alpha, p.beta = 1.f, p.lrelu = lrelu_slope;
    p.a_ld = x_ld, p.out_ld = y_ld, p.in_stride = stride;
    p.batch = batch, p.h = h * stride, p.w = w * stride, p.mh = h, p.mw = w, p.kch = cin, p.nch = cout, p.ncls = 1;
    // K chunks per ring slot: four (eight K16 slices per barrier) where Cin allows it
    p.ntaps = (cin % 128) == 0 ? 4 : (cin % 64) == 0 ? 2 : 1;
    for (int i = 0; i < p.ntaps; ++i) p.taps[i] = i;
    wgmma_conv::tiles(p);
    return E4S_OK;
}

extern "C" int e4s_conv1x1_tcr_f32(const float* x, int x_ld, const void* w_hilo_bf16, const float* bias, float alpha,
                                   const float* r0, const float* r_up, int r_up_ld, float* y, int y_ld, int batch, int h, int w,
                                   int cin, int cout, int stride, float lrelu_slope, void* stream) {
    wgmma_conv::Params p{};
    if (const int rc = pw_params(p, x, x_ld, w_hilo_bf16, bias, alpha, r0, r_up, r_up_ld, y, y_ld, batch, h, w, cin, cout, stride,
                                 lrelu_slope))
        return rc;
    // the N tile (and with it each output's sum order) follows the channel count only: bit identical at any batch
    return wgmma_conv::launch<wgmma_conv::FWD_PW>(p, (cout % 64) == 0 ? 64 : 32, (cudaStream_t)stream);
}

extern "C" int e4s_conv1x1_factor_tcr_f32(const float* x, int x_ld, const void* w_hilo_bf16, const float* bias,
                                          const float* factor, float* y, int y_ld, int batch, int h, int w, int cin, int cout,
                                          void* stream) {
    E4S_REQUIRE(factor, E4S_ERR_ARG);
    wgmma_conv::Params p{};
    if (const int rc = pw_params(p, x, x_ld, w_hilo_bf16, bias, 1.f, nullptr, nullptr, 0, y, y_ld, batch, h, w, cin, cout, 1, 1.f))
        return rc;
    p.factor = factor;
    return wgmma_conv::launch<wgmma_conv::FWD_PWF>(p, (cout % 64) == 0 ? 64 : 32, (cudaStream_t)stream);
}

// The mosaic of a volumetric launch (VolGrid): gutterless stacked slices when the tiles fit them exactly, else cells with
// one-pixel zero gutters, 16 to a mosaic row (16 (W + 1) columns: a whole number of 16-pixel tiles).  Returns the mosaic
// size (rows, columns) in mh, mw.
static wgmma_conv::VolGrid vol_grid(int batch, int depth, int ho, int wo, int& mh, int& mw) {
    using namespace wgmma_conv;
    VolGrid v{};
    v.depth = depth, v.cells = batch * depth;
    v.gutter = (ho % TH) == 0 && (wo % TW) == 0 ? 0 : 1;
    v.ncx = v.gutter ? 16 : 1;
    mh = (int)e4s_ceil_div(v.cells, v.ncx) * (ho + v.gutter), mw = v.ncx * (wo + v.gutter);
    return v;
}

extern "C" int e4s_conv3d_tcr_plan(int batch, int depth, int ho, int wo, int* mosaic_h, int* mosaic_w) {
    E4S_REQUIRE(batch > 0 && depth > 0 && ho > 0 && wo > 0 && mosaic_h && mosaic_w, E4S_ERR_ARG);
    vol_grid(batch, depth, ho, wo, *mosaic_h, *mosaic_w);
    return E4S_OK;
}

// The volumetric entries: x, y channel slices of [B, *, *, D, *] buffers with voxel pitches x_vp, y_vp (floats)
// (r0: added after the bias, before the ReLU, pitched like y, or NULL)
static int conv3d(const float* x, int x_vp, const void* w_hilo_bf16, const float* bias, float* y, int y_vp, int batch, int depth,
                  int h, int w, int cin, int cout, int up, int relu, void* stream, const float* r0 = nullptr) {
    E4S_REQUIRE(x && w_hilo_bf16 && y, E4S_ERR_ARG);
    E4S_REQUIRE(batch > 0 && depth > 0 && h > 0 && w > 0 && cin > 0 && cout > 0 && x_vp >= cin && y_vp >= cout, E4S_ERR_ARG);
    E4S_REQUIRE((cin % 32) == 0 && (cout % 32) == 0, E4S_ERR_SHAPE);
    E4S_REQUIRE((x_vp % 4) == 0 && (y_vp % 4) == 0, E4S_ERR_ALIGN);
    E4S_REQUIRE(e4s_aligned16(x) && e4s_aligned16(w_hilo_bf16) && e4s_aligned16(y) && (!bias || e4s_aligned16(bias)) &&
                    (!r0 || e4s_aligned16(r0)),
                E4S_ERR_ALIGN);
    const int m = up ? 2 : 1;
    // 32-bit index arithmetic inside a sample and the mosaic
    E4S_REQUIRE((int64_t)h * m * w * m * depth * (x_vp > y_vp ? x_vp : y_vp) < (1ll << 31) &&
                    (int64_t)batch * depth * (h * m + 1) * (w * m + 1) < (1ll << 30),
                E4S_ERR_SHAPE);
    wgmma_conv::Params p{};
    p.a = x, p.wt = static_cast<const __nv_bfloat16*>(w_hilo_bf16), p.bias = bias, p.out = y;
    p.alpha = 1.f, p.beta = 1.f, p.lrelu = relu ? 0.f : 1.f, p.residual = r0;
    p.a_ld = depth * x_vp, p.out_ld = depth * y_vp, p.vox_in = x_vp, p.vox_out = y_vp, p.up = up ? 1 : 0;
    p.batch = 1, p.h = h * m, p.w = w * m, p.kch = 3 * cin, p.nch = cout, p.ncls = 1;
    p.vol = vol_grid(batch, depth, h * m, w * m, p.mh, p.mw);
    wgmma_conv::set_taps(p, 0);
    wgmma_conv::tiles(p);
    // the N tile (and with it each output's sum order) follows the channel count only: bit identical at any batch
    return wgmma_conv::launch<wgmma_conv::FWD_VOL>(p, (cout % 64) == 0 ? 64 : 32, (cudaStream_t)stream);
}

extern "C" int e4s_conv3d_tcr_f32(const float* x, const void* w_hilo_bf16, const float* bias, float* y, int batch, int depth,
                                  int h, int w, int cin, int cout, int up, int relu, void* stream) {
    return conv3d(x, cin, w_hilo_bf16, bias, y, cout, batch, depth, h, w, cin, cout, up, relu, stream);
}

extern "C" int e4s_conv3d_pitched_tcr_f32(const float* x, int x_vp, const void* w_hilo_bf16, const float* bias, float* y, int y_vp,
                                          int batch, int depth, int h, int w, int cin, int cout, int up, int relu, void* stream) {
    return conv3d(x, x_vp, w_hilo_bf16, bias, y, y_vp, batch, depth, h, w, cin, cout, up, relu, stream);
}

extern "C" int e4s_conv3d_residual_tcr_f32(const float* x, const void* w_hilo_bf16, const float* bias, const float* residual,
                                           float* y, int batch, int depth, int h, int w, int cin, int cout, int relu, void* stream) {
    E4S_REQUIRE(residual, E4S_ERR_ARG);
    return conv3d(x, cin, w_hilo_bf16, bias, y, cout, batch, depth, h, w, cin, cout, 0, relu, stream, residual);
}

extern "C" int e4s_conv7x7_slices_tcr_f32(const float* x, const void* w_hilo_bf16, float* y, int batch, int depth, int h, int w,
                                          int cin, void* stream) {
    using namespace wgmma_conv;
    E4S_REQUIRE(x && w_hilo_bf16 && y, E4S_ERR_ARG);
    E4S_REQUIRE(batch > 0 && depth > 0 && h > 0 && w > 0 && cin > 0, E4S_ERR_ARG);
    E4S_REQUIRE((cin % KC) == 0 && (h % TH) == 0 && (w % TW) == 0 && batch <= 65535 && depth <= 65535, E4S_ERR_SHAPE);
    E4S_REQUIRE(e4s_aligned16(x) && e4s_aligned16(w_hilo_bf16) && e4s_aligned16(y), E4S_ERR_ALIGN);
    const int tiles_x = w / TW;
    static E4sSmemOptIn optin;
    if (const int rc = e4s_smem_optin(optin, conv7x7_slices_kernel, K7_SMEM)) return rc;
    conv7x7_slices_kernel<<<dim3((unsigned)(tiles_x * (h / TH)), (unsigned)depth, (unsigned)batch), NUM_THREADS, K7_SMEM,
                            (cudaStream_t)stream>>>(x, static_cast<const __nv_bfloat16*>(w_hilo_bf16), y, depth, h, w, cin,
                                                    tiles_x);
    return e4s_launch_status();
}
