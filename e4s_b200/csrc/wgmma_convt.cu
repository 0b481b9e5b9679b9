// The up-sampling layers' transposed-convolution GEMMs on register operands - convt_rs_kernel (unmasked: all four parity
// classes of a pixel tile per work item) and rows_rs_kernel (masked: gathered (pixel, region) rows, one class per work
// item) - and the passes around them: the blur passes and the masked layers' row list.
#include "wgmma_conv.cuh"

namespace wgmma_conv {

// A row of the masked transposed-convolution GEMM: T' pixel (m, n) computed with the style of region r, packed as
// m (14 bits) | n (13 bits) | r (5 bits).
constexpr int ROW_NBITS = 13;
__host__ __device__ constexpr uint32_t row_pack(int m, int n, int r) {
    return ((uint32_t)m << (ROW_NBITS + 5)) | ((uint32_t)n << 5) | (uint32_t)r;
}

__device__ __forceinline__ float4 epilogue4(float4 a, float4 d, float z, float4 bv, int act) {
    float4 o = make_float4(a.x * d.x + (z + bv.x), a.y * d.y + (z + bv.y), a.z * d.z + (z + bv.z), a.w * d.w + (z + bv.w));
    if (act) {
        o.x = lrelu_scaled(o.x, 0.2f, SQRT2);
        o.y = lrelu_scaled(o.y, 0.2f, SQRT2);
        o.z = lrelu_scaled(o.z, 0.2f, SQRT2);
        o.w = lrelu_scaled(o.w, 0.2f, SQRT2);
    }
    return o;
}

// ---- transposed-convolution GEMM on register operands: all four parity classes per work item
// The unmasked layers' T' (see the up-sampling section below) is a stride-1 convolution over the 2 x 2 taps (dy, dx) in
// {0, 1}^2 with N = 4 Cout class-stacked channels, and class (a, c) uses only the taps with (dy || !a) && (dx || !c).
// A work item is 128 rows times one 32-channel slice o0 .. o0 + 31 of Cout in every class: 128 accumulator columns,
// ordered by class [(0,1), (0,0), (1,0), (1,1)].  Then every tap's classes are one contiguous column range - tap (0,0): columns 32-63, (0,1): 0-63,
// (1,0): 32-95, (1,1): 0-127 - and each tap's B tiles are one contiguous block: exactly the 9 class-tap products (ct_mma),
// no zero weights, one halo copy and four A-fragment builds per 32-channel chunk.  The accumulator starts at zero and
// every MMA accumulates, so no class needs a first-MMA flag.  Per element the sum order is chunk, tap (0,0), (0,1), (1,0),
// (1,1) (those the class uses), K16 slice, split product: that of a one-class GEMM over the class's own taps, fixed
// whatever the launch, so the output is bit reproducible.
// The B tiles of a chunk are the 32 x 32 class tiles of the w_convt_hilo planes, copied tap by tap in the column order
// ([w_hi tiles | w_lo tiles] per tap, 9 x 2 x 2 KB = 36 KB).  Resident (RES) when every chunk's 36 KB fit beside the two
// halo slots: copied once per slice (the slice is the outermost item index), else streamed with the chunk's halo.
// Rows: an 8 x 16 pixel tile of the (H + 1) x (W + 1) grid; the halo is its 9 x 17 source pixels (taps {0, 1}^2 only).
// Raw store to T' [B, H+1, W+1, 4 Cout], channel (2a + c) Cout + o.
constexpr int CT_TILE = 32 * KC * 2;                       // one 32 x 32 class tile of one bf16 plane
constexpr int CT_CHUNK = 18 * CT_TILE;                     // a chunk's 9 class tiles, both planes
constexpr int CT_HW = TW + 1, CT_HPIX = (TH + 1) * CT_HW;  // pixel-tile halo: 9 x 17
// tap k = 2 dy + dx: first column slot (of 32), slots, first tile of its weights in the chunk block
__host__ __device__ constexpr int ct_slot0(int k) { return k == 1 ? 0 : k == 3 ? 0 : 1; }
__host__ __device__ constexpr int ct_nslot(int k) { return k == 0 ? 1 : k == 3 ? 4 : 2; }
__host__ __device__ constexpr int ct_tile0(int k) { return k == 0 ? 0 : k == 1 ? 2 : k == 2 ? 6 : 10; }
__host__ __device__ constexpr int ct_class(int slot) { return slot == 0 ? 1 : slot == 1 ? 0 : slot; }

// The split products of one tap and K16 slice on its NS column slots from slot S0 (accumulator registers 16 S0 ..), B
// from bh (w_hi tiles; w_lo tiles follow): one m64n32k16 MMA per slot.  (Wider MMAs over the tap's whole column range
// would need fewer instructions, but ptxas serialises every wgmma of the kernel when register subsets of different
// widths or offsets overlap - C7511, "insufficient register resources for the wgmma pipeline"; 32-column MMAs on the four
// disjoint slots stay pipelined.)
template <int S0, int NS>
__device__ __forceinline__ void ct_mma(float (&acc)[64], const uint32_t (&hi)[4], const uint32_t (&lo)[4], uint32_t bh) {
#pragma unroll
    for (int i = 0; i < NS; ++i) {
        float (&d)[16] = *reinterpret_cast<float(*)[16]>(&acc[16 * (S0 + i)]);
        const uint32_t b = bh + i * CT_TILE;
        wgmma(d, lo, b, 1);
        wgmma(d, hi, b + NS * CT_TILE, 1);
        wgmma(d, hi, b, 1);
    }
}

template <bool RES>
__global__ void __launch_bounds__(NUM_THREADS, 1) convt_rs_kernel(const __grid_constant__ Params prm, const int items, const int stage) {
    // (read through a reference: the parameter read directly gives the same instructions, two of them in another order)
    const Params& p = prm;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~uintptr_t(127));
    const uint32_t smem_s = (uint32_t)__cvta_generic_to_shared(smem);
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5, g = lane >> 2, q = lane & 3, hc = t & 7;
    const int H = p.h, W = p.w, cout = p.nch / 4, nchunks = p.kch / KC, plane = p.nch * p.kch;
    const int halo_bytes = RES ? stage : stage - CT_CHUNK;
    const uint32_t w_s = smem_s + 2 * stage;              // resident weight block: chunk kc at w_s + kc * CT_CHUNK

    // work item: pixel tile (tx, ty), sample b, slice n0 .. n0 + 31 of Cout (the outermost index)
    auto decode = [&](int idx) { return decode_item<false>(p, idx, 32); };
    // this thread's fragment rows g, g + 8 of tile row `warp`: halo offsets of their tap (0,0) source pixels
    const int hb[2] = {warp * CT_HW + g, warp * CT_HW + g + 8};
    // this thread's styles of chunk kc: its fragment channels (one style per sample)
    auto load_styles = [&](const Item& it, int kc, float2 (&sv)[4]) {
#pragma unroll
        for (int j = 0; j < 4; ++j) sv[j] = __ldg(reinterpret_cast<const float2*>(p.s + it.b * p.kch + kc * KC + 8 * j + 2 * q));
    };
    // the 18 (class tile, plane) pairs of chunk kc of slice o0 at dst: copy e of the chunk is pair e / 128, row
    // 8 (c / 32) + c % 8 and channel quad (c / 8) % 4 of the tile (c = e % 128), byte 16 c of the tile
    auto copy_weights = [&](int o0, int kc, uint32_t dst) {
#pragma unroll
        for (int i = 0; i < 18 * 128 / NUM_THREADS; ++i) {
            const int e = t + NUM_THREADS * i, u = e >> 7, c = e & 127;
            const int k = u < 2 ? 0 : u < 6 ? 1 : u < 10 ? 2 : 3, ns = ct_nslot(k), w = u - ct_tile0(k);
            const int hl = w >= ns, cls = ct_class(ct_slot0(k) + w - hl * ns);
            const int n = cls * cout + o0 + (c >> 5) * 8 + (c & 7);
            cp_async16(dst + e * 16, p.wt + (hl * 9 + (k >> 1) * 3 + (k & 1)) * plane + n * p.kch + kc * KC + ((c >> 3) & 3) * 8, 16);
        }
    };
    auto copy_block = [&](int o0) {
#pragma unroll 1
        for (int kc = 0; kc < nchunks; ++kc) copy_weights(o0, kc, w_s + kc * CT_CHUNK);
    };
    // ring slot buf <- chunk kc of the item's halo (zero outside the image) and, streaming, its weights
    auto prefetch = [&](const Item& it, int kc, int buf) {
        const uint32_t st = smem_s + buf * stage;
        const float* xb = p.a + (int64_t)it.b * H * W * p.kch + kc * KC + hc * 4;
        const int sy0 = it.ty * TH - 1, sx0 = it.tx * TW - 1;
#pragma unroll
        for (int i = 0; i < (CT_HPIX * 8 + NUM_THREADS - 1) / NUM_THREADS; ++i) {
            const int hp = (t >> 3) + 32 * i;
            if (hp < CT_HPIX) {
                const int hy = hp / CT_HW, sy = sy0 + hy, sx = sx0 + hp - hy * CT_HW;
                const bool ok = sy >= 0 && sy < H && sx >= 0 && sx < W;
                cp_async16(tile_at(st, hp, hc), ok ? xb + (sy * W + sx) * p.kch : p.a, ok ? 16 : 0);
            }
        }
        if (!RES) copy_weights(it.n0, kc, st + halo_bytes);
        cp_async_commit();
    };

    float acc[64];
    uint32_t fh[2][2][4], fl[2][2][4];                    // [tap % 2][K16 slice][register]: x_hi, x_lo fragments
    // a tap's fragments: this thread's rows at halo offset toff from their tap (0,0) pixels
    auto build = [&](const uint8_t* halo, int toff, const float2 (&sv)[4], uint32_t (&hi)[2][4], uint32_t (&lo)[2][4]) {
        auto hp = [&](int h) { return hb[h] + toff; };
#pragma unroll
        for (int ks = 0; ks < 2; ++ks) build_frag(halo, hp, q, ks, hi[ks], lo[ks], sv, sv);
    };
    // tap K's MMAs, both K16 slices, B from bt (its tiles in the chunk block)
    auto issue = [&](auto kk, uint32_t bt, uint32_t (&hi)[2][4], uint32_t (&lo)[2][4]) {
        constexpr int K = decltype(kk)::value;
        fence_regs(acc);
        fence_frag(hi);
        fence_frag(lo);
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < 2; ++ks) ct_mma<ct_slot0(K), ct_nslot(K)>(acc, hi[ks], lo[ks], bt + ct_tile0(K) * CT_TILE + ks * 2 * LBO);
        wgmma_commit();
        fence_regs(acc);
        fence_frag(hi);
        fence_frag(lo);
    };
    auto store_item = [&](const Item& it) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int iy = it.ty * TH + warp, ix = it.tx * TW + g + 8 * h;
            if (iy > H || ix > W) continue;
            float* dst = p.out + (((int64_t)it.b * (H + 1) + iy) * (W + 1) + ix) * p.nch;
#pragma unroll
            for (int nf = 0; nf < 16; ++nf)
                *reinterpret_cast<float2*>(dst + ct_class(nf >> 2) * cout + it.n0 + (nf & 3) * 8 + 2 * q) =
                    make_float2(acc[4 * nf + 2 * h], acc[4 * nf + 2 * h + 1]);
        }
    };

    int item = blockIdx.x;
    if (item >= items) return;
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    Item cur = decode(item), nxt;
    float2 sty[4], sty_n[4];
    load_styles(cur, 0, sty);
    int kc = 0, buf = 0;
    if (RES) copy_block(cur.n0);                          // committed with the first halo
    prefetch(cur, 0, 0);
#pragma unroll 1
    while (true) {
        const bool last_chunk = kc == nchunks - 1;
        const int item_n = last_chunk ? item + (int)gridDim.x : item, kc_n = last_chunk ? 0 : kc + 1;
        const bool more = item_n < items;
        // slot buf complete and visible to the async proxy; every MMA of the previous chunk retired (wait_group 0 below),
        // so the other slot may be refilled once this chunk's first MMAs are issued.  Fragment set k % 2 is rebuilt
        // after wait_group 1 has retired tap k - 2, its last reader.
        cp_async_wait_all();
        fence_proxy_async();
        __syncthreads();
        const uint8_t* halo = smem + buf * stage;
        const uint32_t bt = RES ? w_s + kc * CT_CHUNK : smem_s + buf * stage + halo_bytes;
        build(halo, 0, sty, fh[0], fl[0]);
        issue(std::integral_constant<int, 0>{}, bt, fh[0], fl[0]);
        if (more) {                                       // while tap (0,0)'s MMAs run
            nxt = last_chunk ? decode(item_n) : cur;
            prefetch(nxt, kc_n, buf ^ 1);
            load_styles(nxt, kc_n, sty_n);
        }
        build(halo, 1, sty, fh[1], fl[1]);
        issue(std::integral_constant<int, 1>{}, bt, fh[1], fl[1]);
        wgmma_wait<1>();
        build(halo, CT_HW, sty, fh[0], fl[0]);
        issue(std::integral_constant<int, 2>{}, bt, fh[0], fl[0]);
        wgmma_wait<1>();
        build(halo, CT_HW + 1, sty, fh[1], fl[1]);
        issue(std::integral_constant<int, 3>{}, bt, fh[1], fl[1]);
        wgmma_wait<0>();
        fence_regs(acc);
        if (RES && more && nxt.n0 != cur.n0) {            // next slice: its block, once both warpgroups' MMAs retired;
            __syncthreads();                              // the barrier at the top of the loop waits for the copies
            copy_block(nxt.n0);
            cp_async_commit();
        }
        if (last_chunk) {
            store_item(cur);
#pragma unroll
            for (int i = 0; i < 64; ++i) acc[i] = 0.f;
        }
        if (!more) break;
        cur = nxt, item = item_n, kc = kc_n, buf ^= 1;
#pragma unroll
        for (int j = 0; j < 4; ++j) sty[j] = sty_n[j];
    }
}

// ---- masked transposed-convolution GEMM on register operands (rows_rs_kernel): gathered rows, one parity class per work item
// The masked layers' T' rows are (T' pixel, region) pairs from a row list (p.rows, see the masked up-sampling section
// below), so there is no pixel tile to share a halo.  A work item is one 128-row block rb of sample b's list times NT
// channels n0 .. of ONE class cls (columns cls Cout + ..): K runs over the class's taps in the order {0, 1, 3, 4} (those
// it uses: 4 >> popcount(cls) of them) and, inside each tap, the 32-channel chunks - tap-outer, chunk-inner.  A K step
// (tap, chunk) stages the 128 rows' source pixels at the tap's offset (16-byte cp.async copies, zero off the grid and past
// the list's end; an A tile, tile_at) and the step's NT x 32 weight tiles; each consumer thread builds its
// fragment rows from them scaled by the style of the row's own region (read per step from the style table), splits them
// (split2) and issues split_mma.  Per element the sum order is tap, chunk, K16 slice, split product - whatever NT is
// (64 and 128 give the same bits), so a face's output does not depend on the batch it is in.
// A slot of the two-slot cp.async ring holds p.ntaps consecutive K steps ([A tiles | B tiles]); the ring runs over the
// flattened (item, step group) sequence, one barrier per group, and the fragments are double-buffered across steps as in
// conv3x3_rs_kernel.
// Schedule: the items of the launch are those of the row blocks holding rows (blocks past a sample's row count, and every
// block of a sample whose list overflowed, row_count > cap, have none), in the order sample, row block, class, slice.
// Every row block carries the same 9 nchunks Cout / NT K steps, so each CTA computes from the row counts where its equal
// share of the launch's steps begins and ends and takes the items that start inside it: the chains of 4, 2, 2 and 1 taps
// balance over the CTAs, and a CTA runs all classes of a row block back to back, sharing its gathered rows in L2.  Raw
// store to T'c [B, cap, 4 Cout] (rows below the count).
struct RowItem {
    int b, rb, cls, n0, cnt, nsteps;
};
// item k (class k / slices, slice k % slices) of row block rb of sample b, starting at step s of the launch
struct RowPos {
    int b, rb, k;
    int64_t s;
};
template <int NT>
__global__ void __launch_bounds__(NUM_THREADS, 1) rows_rs_kernel(const __grid_constant__ Params p, int, const int stage) {
    constexpr int A_TILE = M * KC * 4, B_PLANE = NT * KC * 2, B_CP = B_PLANE / 16;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~uintptr_t(127));
    const uint32_t smem_s = (uint32_t)__cvta_generic_to_shared(smem);
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5, g = lane >> 2, q = lane & 3, hc = t & 7;
    const int H = p.h, W = p.w, cout = p.nch / 4, nchunks = p.kch / KC, plane = p.nch * p.kch, spg = p.ntaps;
    const int w_ofs = spg * A_TILE;                       // B tiles of a slot: step k at w_ofs + 2 k B_PLANE

    const int nsl = p.n_tiles;
    // row blocks of sample b holding rows
    auto blocks_of = [&](int b) {
        const int c = __ldg(p.row_count + b);
        return c <= p.cap ? (c + M - 1) / M : 0;
    };
    // this CTA's share [lo, hi) of the launch's K steps
    int64_t nblk = 0;
    for (int b = 0; b < p.batch; ++b) nblk += blocks_of(b);
    const int64_t per_block = 9ll * nchunks * nsl, total = nblk * per_block;
    const int64_t lo = total * blockIdx.x / gridDim.x, hi = total * (blockIdx.x + 1) / gridDim.x;
    auto decode = [&](const RowPos& q) {
        RowItem it;
        it.b = q.b, it.rb = q.rb, it.cls = q.k / nsl;
        it.n0 = it.cls * cout + (q.k - it.cls * nsl) * NT;
        it.cnt = __ldg(p.row_count + q.b);
        it.nsteps = (4 >> __popc(it.cls)) * nchunks;
        return it;
    };
    // the item after q: next slice, class, row block holding rows, sample
    auto advance = [&](RowPos q) {
        q.s += (4 >> __popc(q.k / nsl)) * nchunks;
        if (++q.k == 4 * nsl) {
            q.k = 0;
            if (++q.rb == blocks_of(q.b)) {
                q.rb = 0;
                do ++q.b;
                while (q.b < p.batch && blocks_of(q.b) == 0);
            }
        }
        return q;
    };
    auto mine = [&](const RowPos& q) { return q.b < p.batch && q.s < hi; };
    // K step s of the item: tap ti = s / nchunks of its class (offset (dy, dx)), chunk s % nchunks
    auto step_tap = [&](const RowItem& it, int s, int& dy, int& dx) {
        const int ti = s / nchunks;
        if (it.cls & 2) dy = 1, dx = (it.cls & 1) ? 1 : ti;
        else if (it.cls & 1) dy = ti, dx = 1;
        else dy = ti >> 1, dx = ti & 1;
    };
    // the item's rows this thread gathers, (t >> 3) + 32 i: packed positions, valid where i < vcnt (loaded once per item,
    // before its first copies)
    uint32_t rv[4];
    int vcnt = 0;
    // ring slot buf <- step group gi of the item: per step the gathered rows (row r at r * 128 bytes) and both weight planes
    auto prefetch = [&](const RowItem& it, int gi, int buf) {
        if (gi == 0) {
            vcnt = 0;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int r = it.rb * M + (t >> 3) + 32 * i;
                rv[i] = r < it.cnt ? __ldg(p.rows + (int64_t)it.b * p.cap + r) : 0u;
                vcnt += r < it.cnt;
            }
        }
        const uint32_t st = smem_s + buf * stage;
        const int s0 = gi * spg, ns = min(spg, it.nsteps - s0);
        for (int k = 0; k < ns; ++k) {
            const int s = s0 + k, kc = s % nchunks;
            int dy, dx;
            step_tap(it, s, dy, dx);
            const float* xb = p.a + (int64_t)it.b * H * W * p.kch + kc * KC + hc * 4;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int r = (t >> 3) + 32 * i;
                const int sy = (int)(rv[i] >> (ROW_NBITS + 5)) + dy - 1, sx = (int)((rv[i] >> 5) & ((1u << ROW_NBITS) - 1)) + dx - 1;
                const bool ok = i < vcnt && sy >= 0 && sy < H && sx >= 0 && sx < W;
                cp_async16(tile_at(st + k * A_TILE, r, hc), ok ? xb + (sy * W + sx) * p.kch : p.a, ok ? 16 : 0);
            }
            // copy c of a plane: row 8 (c / 32) + c % 8, channel quad (c / 8) % 4 of the tile, byte 16 c
            const int tap = dy * 3 + dx;
            const uint32_t bd = st + w_ofs + k * 2 * B_PLANE;
#pragma unroll
            for (int c = t; c < B_CP; c += NUM_THREADS) {
                const __nv_bfloat16* wb = p.wt + (it.n0 + (c >> 5) * 8 + (c & 7)) * p.kch + kc * KC + ((c >> 3) & 3) * 8;
                cp_async16(bd + c * 16, wb + tap * plane, 16);
                cp_async16(bd + B_PLANE + c * 16, wb + (9 + tap) * plane, 16);
            }
        }
        cp_async_commit();
    };
    // regions of this thread's fragment rows 16 warp + g, + 8
    auto row_regions = [&](const RowItem& it, int (&c)[2]) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int i = it.rb * M + warp * 16 + g + 8 * h;
            c[h] = i < it.cnt ? min((int)(__ldg(p.rows + (int64_t)it.b * p.cap + i) & 31u), p.ncls - 1) : 0;
        }
    };
    // styles of step s's chunk at this thread's fragment channels, per fragment row's region
    auto load_styles = [&](const RowItem& it, const int (&c)[2], int s, float2 (&sv)[2][4]) {
        const int kc = s % nchunks;
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int j = 0; j < 4; ++j)
                sv[h][j] = __ldg(reinterpret_cast<const float2*>(p.s + (it.b * p.ncls + c[h]) * p.kch + kc * KC + 8 * j + 2 * q));
    };

    SplitAcc<NT> acc{};                                   // zero: the fences read every register
    uint32_t fh[2][2][4], fl[2][2][4];                    // [step % 2][K16 slice][register]: x_hi, x_lo fragments
    // a step's fragments from its A tile: this thread's rows 16 warp + g, + 8 of the block
    auto build = [&](const uint8_t* a, const float2 (&sv)[2][4], uint32_t (&hi)[2][4], uint32_t (&lo)[2][4]) {
        auto hp = [&](int h) { return warp * 16 + g + 8 * h; };
#pragma unroll
        for (int ks = 0; ks < 2; ++ks) build_frag(a, hp, q, ks, hi[ks], lo[ks], sv[0], sv[1]);
    };
    auto store_item = [&](const RowItem& it) {
        acc.fold();
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int i = it.rb * M + warp * 16 + g + 8 * h;
            if (i >= it.cnt) continue;
            float* dst = p.out + ((int64_t)it.b * p.cap + i) * p.nch + it.n0 + 2 * q;
#pragma unroll
            for (int nf = 0; nf < NT / 8; ++nf)
                *reinterpret_cast<float2*>(dst + nf * 8) = make_float2(acc.d[4 * nf + 2 * h], acc.d[4 * nf + 2 * h + 1]);
        }
    };

    // the first item starting at or after lo: in row block lo / per_block (the n-th holding rows), else the next one
    RowPos pos{0, 0, 0, lo - lo % per_block};
    for (int64_t n = lo / per_block; pos.b < p.batch; ++pos.b) {
        const int nb = blocks_of(pos.b);
        if (n < nb) {
            pos.rb = (int)n;
            break;
        }
        n -= nb;
    }
    while (pos.s < lo) pos = advance(pos);
    if (!mine(pos)) return;
    RowPos pos_n = advance(pos);
    RowItem cur = decode(pos), nxt;
    int cls[2], cls_n[2];
    row_regions(cur, cls);
    float2 sty[2][4];                                     // styles of the next step to build
    load_styles(cur, cls, 0, sty);
    int gi = 0, buf = 0;
    prefetch(cur, 0, 0);
#pragma unroll 1
    while (true) {
        const bool last_group = (gi + 1) * spg >= cur.nsteps;
        const int gi_n = last_group ? 0 : gi + 1;
        const bool more = !last_group || mine(pos_n);
        // slot buf complete and visible to the async proxy; every MMA of the previous group retired (wait_group 0 below),
        // so the other slot may be refilled once this group's first MMAs are issued.  Fragment set k % 2 is rebuilt
        // after wait_group 1 has retired step k - 2, its last reader.
        cp_async_wait_all();
        fence_proxy_async();
        __syncthreads();
        const uint8_t* a_slot = smem + buf * stage;
        const uint32_t b_slot = smem_s + buf * stage + w_ofs;
        const int s0 = gi * spg, ns = min(spg, cur.nsteps - s0);
#pragma unroll 1
        for (int k = 0; k < ns; k += 2) {
            if (k >= 2) wgmma_wait<1>();
            build(a_slot + k * A_TILE, sty, fh[0], fl[0]);
            if (s0 + k + 1 < cur.nsteps) load_styles(cur, cls, s0 + k + 1, sty);
            issue_rs(acc, fh[0], fl[0], b_slot + k * 2 * B_PLANE, s0 + k == 0);
            if (k + 1 < ns) {
                wgmma_wait<1>();
                build(a_slot + (k + 1) * A_TILE, sty, fh[1], fl[1]);
                if (s0 + k + 2 < cur.nsteps) load_styles(cur, cls, s0 + k + 2, sty);
                issue_rs(acc, fh[1], fl[1], b_slot + (k + 1) * 2 * B_PLANE, false);
            }
            if (k == 0 && more) {                         // once the group's first two steps are queued
                if (last_group) {
                    nxt = decode(pos_n);
                    row_regions(nxt, cls_n);
                } else {
                    nxt = cur, cls_n[0] = cls[0], cls_n[1] = cls[1];
                }
                prefetch(nxt, gi_n, buf ^ 1);
            }
        }
        wgmma_wait<0>();
        acc.fence();
        if (last_group) store_item(cur);
        if (!more) break;
        if (last_group) {
            cur = nxt, cls[0] = cls_n[0], cls[1] = cls_n[1];
            pos_n = advance(pos_n);
            load_styles(cur, cls, 0, sty);
        }
        gi = gi_n, buf ^= 1;
    }
}

// ------------------------------------------------------------------------------------------ host
// The unmasked transposed-convolution GEMM (convt_rs_kernel), persistent, one CTA per SM.
static int launch_convt(const Params& p, int64_t items, cudaStream_t st) {
    if (items >= (1ll << 31) - 1024 || (int64_t)p.h * p.w * p.kch >= (1ll << 31) || 18ll * p.nch * p.kch >= (1ll << 31))
        return E4S_ERR_SHAPE;
    // the weights stay resident when every chunk's class tiles fit beside the two halo slots; E4S_B200_RS_STREAM=1
    // streams them with every chunk regardless (tests)
    const int halo = CT_HPIX * KC * 4;
    const int64_t block = (int64_t)(p.kch / KC) * CT_CHUNK;
    const char* f = getenv("E4S_B200_RS_STREAM");
    const bool resident = !(f && atoi(f) != 0) && 128 + 2 * halo + block <= e4s_smem_optin_limit();
    const int stage = resident ? halo : halo + CT_CHUNK;
    const size_t smem = 128 + 2 * (size_t)stage + (resident ? (size_t)block : 0);
    static E4sSmemOptIn optin[2];
    auto kernel = resident ? convt_rs_kernel<true> : convt_rs_kernel<false>;
    if (const int rc = e4s_smem_optin(optin[resident], kernel, smem)) return rc;
    const int64_t grid = items < num_sms() ? items : num_sms();
    kernel<<<(unsigned)grid, NUM_THREADS, smem, st>>>(p, (int)items, stage);
    return e4s_launch_status();
}

// N-tile width of the gathered-row GEMM (one class of Cout channels per item): 128 when Cout allows it and the items at
// that width (row blocks x 4 classes x Cout / 128, counted to the cap) fill the SMs twice, else 64 where Cout allows it,
// else 32.  64 and 128 give the same bits; the stacked 32-channel form is taken only where 64 does not divide Cout, so the
// width never changes a result.  E4S_B200_RS_NTILE=64|128 forces a width Cout allows (tests).
static int pick_ntile_rows(int cout, int64_t row_blocks) {
    const char* f = getenv("E4S_B200_RS_NTILE");
    const int v = f ? atoi(f) : 0;
    if ((v == 64 || v == 128) && cout % v == 0) return v;
    if (cout % 128 == 0 && row_blocks * 4 * (cout / 128) >= 2 * num_sms()) return 128;
    return cout % 64 == 0 ? 64 : 32;
}

// The masked transposed-convolution GEMM (rows_rs_kernel), persistent: p.tiles_x row blocks per sample,
// p.n_tiles = Cout / nt slices per class.  A ring slot holds up to four K steps (p.ntaps), as many as two slots fit.
template <int NT>
static int launch_rows(Params p, cudaStream_t st) {
    p.n_tiles = p.nch / 4 / NT;
    const int64_t items = (int64_t)p.tiles_x * p.batch * 4 * p.n_tiles;
    if (items >= (1ll << 31) - 1024 || (int64_t)p.h * p.w * p.kch >= (1ll << 31) || 18ll * p.nch * p.kch >= (1ll << 31))
        return E4S_ERR_SHAPE;
    // p.ntaps: K steps per ring slot (this kernel has no tap list; the taps follow the class), as many as two slots fit
    const int step = M * KC * 4 + 2 * NT * KC * 2;        // gathered rows + both weight planes
    p.ntaps = (e4s_smem_optin_limit() - 128) / (2 * step);
    if (p.ntaps > 4) p.ntaps = 4;
    if (p.ntaps < 1) return E4S_ERR_SHAPE;
    const int stage = p.ntaps * step;
    const size_t smem = 128 + 2 * (size_t)stage;
    static E4sSmemOptIn optin;
    auto kernel = rows_rs_kernel<NT>;
    if (const int rc = e4s_smem_optin(optin, kernel, smem)) return rc;
    const int64_t grid = items < num_sms() ? items : num_sms();
    kernel<<<(unsigned)grid, NUM_THREADS, smem, st>>>(p, (int)items, stage);
    return e4s_launch_status();
}

// ---- unmasked up-sampling layer: transposed-convolution GEMM + blur pass
// The stride-2 transposed convolution u[p] = sum_i x[i] w[p - 2 i] (per axis) is stored space-to-depth on a row grid one
// pixel larger than the input: T'[m, n, (a, c), o] = u[2m + a, 2n + c, o] for m <= H, n <= W.  Along an axis, parity a = 0
// takes the taps d = 0 (weight row 2) and d = 1 (row 0) of the source rows m - 1 + d, parity a = 1 only d = 1 (row 1).  So
// it is a stride-1 convolution over the 2 x 2 taps {0, 1, 3, 4} with N = 4 Cout class-stacked channels, and class (a, c)
// uses 4, 2, 2 or 1 of those taps: 9 tap products per input pixel, all four classes in one work item of
// convt_rs_kernel.  The gathered-row GEMM of the masked layers (rows_rs_kernel) has one class per work item
// instead, over that class's own taps.

constexpr int BLUR_ROWS = 32;                         // output rows per thread of the blur pass
constexpr int BLUR_THREADS = 256;

// y[Y, X, o] = act(demod[o] * sum_{p,q} fir[3-p][3-q] T[Y-1+p][X-1+q] + noise_w * noise[Y, X] + bias[o]), the true 4 x 4
// convolution (pad 1) of T = the transposed-convolution output, T[u, v] = T'[u >> 1, v >> 1, (u & 1, v & 1)], zero
// outside 0 <= u <= 2H + 1.  A thread owns 4 channels of the output columns 2j, 2j + 1 over BLUR_ROWS rows and walks down
// T one row at a time: the row's five float4 (T columns 2j - 1 .. 2j + 3) feed the four output rows it touches, and the
// row it completes is stored.  Every output sums p = 0..3, q = 0..3 in that order: the result does not depend on the
// thread layout.
__global__ void __launch_bounds__(BLUR_THREADS, 3) convt_blur_kernel(const float* __restrict__ t, const float* __restrict__ fir,
                                                                  const float* __restrict__ demod,
                                                                  const float* __restrict__ noise,
                                                                  const float* __restrict__ noise_w,
                                                                  const float* __restrict__ bias, float* __restrict__ y,
                                                                  int batch, int h, int w, int cout, int noise_b, int act,
                                                                  int strips) {
    const int cq = cout >> 2;
    int64_t gid = (int64_t)blockIdx.x * BLUR_THREADS + threadIdx.x;
    if (gid >= (int64_t)batch * strips * w * cq) return;
    const int o = (int)(gid % cq) * 4;
    gid /= cq;
    const int j = (int)(gid % w);
    gid /= w;
    const int y0 = (int)(gid % strips) * BLUR_ROWS, b = (int)(gid / strips);
    const int Ho = 2 * h, Wo = 2 * w;
    float f[4][4];
#pragma unroll
    for (int q = 0; q < 16; ++q) f[q >> 2][q & 3] = __ldg(fir + 15 - q);
    const float4 d = demod ? ld4(demod + (int64_t)b * cout + o) : make_float4(1.f, 1.f, 1.f, 1.f);
    const float4 bv = bias ? ld4(bias + o) : make_float4(0.f, 0.f, 0.f, 0.f);
    const float nw = (noise && noise_w) ? __ldg(noise_w) : 0.f;
    const int64_t trow = (int64_t)(w + 1) * 4 * cout;                   // floats per T' row
    const float* tb = t + (int64_t)b * (h + 1) * trow + o;
    // acc[i]: output row Y = u - 2 + i, which T row u reaches through FIR row p = 3 - i
    float4 acc[4][2];
#pragma unroll
    for (int i = 0; i < 4; ++i) acc[i][0] = acc[i][1] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 4
    for (int r = 0; r < BLUR_ROWS + 3; ++r) {
        const int u = y0 - 1 + r;
        float4 v[5];
#pragma unroll
        for (int k = 0; k < 5; ++k) v[k] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (u >= 0 && (u >> 1) <= h) {
            // T column 2j - 1 + k: T' pixel j + ((k - 1) >> 1), class column (k + 1) & 1
            const float* row = tb + (int64_t)(u >> 1) * trow + (int64_t)((u & 1) * 2) * cout + (int64_t)j * 4 * cout;
            if (j > 0) v[0] = ld4(row - 3 * cout);
            v[1] = ld4(row);
            v[2] = ld4(row + cout);
            v[3] = ld4(row + 4 * cout);
            v[4] = ld4(row + 5 * cout);
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int p = 3 - i;
#pragma unroll
            for (int cx = 0; cx < 2; ++cx) {
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const float c = f[p][q];
                    const float4 e = v[cx + q];
                    float4& a = acc[i][cx];
                    a.x = fmaf(c, e.x, a.x), a.y = fmaf(c, e.y, a.y), a.z = fmaf(c, e.z, a.z), a.w = fmaf(c, e.w, a.w);
                }
            }
        }
        const int yo = u - 2;                         // complete: its p = 3 row was this one
        if (r >= 3 && yo < Ho) {
#pragma unroll
            for (int cx = 0; cx < 2; ++cx) {
                const int xo = 2 * j + cx;
                const float z = noise ? nw * __ldg(noise + ((int64_t)(noise_b == 1 ? 0 : b) * Ho + yo) * Wo + xo) : 0.f;
                *reinterpret_cast<float4*>(y + (((int64_t)b * Ho + yo) * Wo + xo) * cout + o) = epilogue4(acc[0][cx], d, z, bv, act);
            }
        }
#pragma unroll
        for (int i = 0; i < 3; ++i) acc[i][0] = acc[i + 1][0], acc[i][1] = acc[i + 1][1];
        acc[3][0] = acc[3][1] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
}

// ---- masked up-sampling layer: transposed-convolution GEMM over (T' pixel, region) rows + region-aware blur pass
// Through the 4 x 4 blur, T' pixel (m, n) (T rows 2m, 2m + 1) reaches only the output pixels Y in [2m - 2, 2m + 2],
// X in [2n - 2, 2n + 2].  It is computed once with the style of each region present in that (clipped) window and for no
// other region; an output pixel of region r reads the rows of its own region, which its window always holds.

constexpr int LIST_THREADS = 1024;
constexpr int BLUR_PIX = 4;                           // output pixels per thread of the masked blur pass

// One block per sample.  need[b, m, n]: the regions of the 5 x 5 window; base[b, m, n]: exclusive prefix sum of their
// counts in row-major (m, n) order; rows[b, base + k]: (m, n, k-th region of need) for rows below cap; count[b]: the
// sample's total (the list is complete only when count <= cap; past cap, count is only known to exceed it).
__global__ void __launch_bounds__(LIST_THREADS) convt_row_list_kernel(const uint8_t* __restrict__ label, uint32_t* __restrict__ need,
                                                                      int* __restrict__ base, int* __restrict__ count,
                                                                      uint32_t* __restrict__ rows, int h, int w, int ncls, int cap) {
    __shared__ int warp_sum[LIST_THREADS / 32];
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5, b = blockIdx.x;
    const int Ho = 2 * h, Wo = 2 * w, npix = (h + 1) * (w + 1);
    const uint8_t* lb = label + (int64_t)b * Ho * Wo;
    int running = 0;
    for (int start = 0; start < npix; start += LIST_THREADS) {
        const int pix = start + t, m = pix / (w + 1), n = pix % (w + 1);
        uint32_t bits = 0;
        if (pix < npix) {
            for (int Y = max(2 * m - 2, 0); Y <= min(2 * m + 2, Ho - 1); ++Y)
                for (int X = max(2 * n - 2, 0); X <= min(2 * n + 2, Wo - 1); ++X)
                    bits |= 1u << region(lb, ncls, Y * Wo + X);
        }
        const int c = __popc(bits);
        int incl = c;                                 // block-wide inclusive scan: within the warp, then over warps
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int v = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += v;
        }
        if (lane == 31) warp_sum[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            int s = warp_sum[lane];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int v = __shfl_up_sync(0xffffffffu, s, o);
                if (lane >= o) s += v;
            }
            warp_sum[lane] = s;
        }
        __syncthreads();
        const int excl = running + (warp ? warp_sum[warp - 1] : 0) + incl - c;
        if (pix < npix) {
            const int64_t gp = (int64_t)b * npix + pix;
            need[gp] = bits;
            base[gp] = excl;
            int i = excl;
            for (uint32_t rb = bits; rb && i < cap; rb &= rb - 1, ++i) rows[(int64_t)b * cap + i] = row_pack(m, n, __ffs(rb) - 1);
        }
        running += warp_sum[LIST_THREADS / 32 - 1];
        __syncthreads();                              // warp_sum is rewritten by the next chunk
        if (running > cap) break;                     // the sample falls back: its list is not read
    }
    if (t == 0) count[b] = running;
}

// y[Y, X, o] = act(demod[r, o] * sum_{p,q} fir[3-p][3-q] T_r[Y-1+p][X-1+q] + noise_w * noise[Y, X] + bias[o]) with
// r = label[Y, X] and T_r the transposed-convolution output computed with region r's style: T_r[u, v] is channel
// ((u & 1, v & 1), o) of compacted row base[m, n] + popcount(need[m, n] & ((1 << r) - 1)), (m, n) = (u >> 1, v >> 1); zero
// for u < 0 or v < 0.  A thread owns 4 channels of BLUR_PIX output pixels along X; p = 0..3, q = 0..3 are summed in that
// order.
// Samples whose list overflowed (count > cap) are left to the folded kernel.
__global__ void __launch_bounds__(BLUR_THREADS) convt_blur_masked_kernel(
    const float* __restrict__ tc, const uint32_t* __restrict__ need, const int* __restrict__ base, const int* __restrict__ count,
    const uint8_t* __restrict__ label, const float* __restrict__ fir, const float* __restrict__ demod,
    const float* __restrict__ noise, const float* __restrict__ noise_w, const float* __restrict__ bias, float* __restrict__ y,
    int batch, int h, int w, int cout, int ncls, int cap, int noise_b, int act) {
    const int cq = cout >> 2, Ho = 2 * h, Wo = 2 * w, xg = (Wo + BLUR_PIX - 1) / BLUR_PIX;
    int64_t gid = (int64_t)blockIdx.x * BLUR_THREADS + threadIdx.x;
    if (gid >= (int64_t)batch * Ho * xg * cq) return;
    const int o = (int)(gid % cq) * 4;
    gid /= cq;
    const int X0 = (int)(gid % xg) * BLUR_PIX;
    gid /= xg;
    const int Y = (int)(gid % Ho), b = (int)(gid / Ho);
    if (__ldg(count + b) > cap) return;
#pragma unroll 1
    for (int X = X0; X < min(X0 + BLUR_PIX, Wo); ++X) {
        const int r = region(label, ncls, ((int64_t)b * Ho + Y) * Wo + X);
        const uint32_t below = (1u << r) - 1u;
        const int64_t pix0 = (int64_t)b * (h + 1) * (w + 1);
        const float* tb = tc + (int64_t)b * cap * 4 * cout + o;
        // T rows Y - 1 .. Y + 2 lie in T' rows m0 + (p + ey) / 2 (2 of them for odd Y, 3 for even Y); the same along x.  All
        // lookups, then all loads, are issued before the first is used.
        const int m0 = (Y - 1) >> 1, n0 = (X - 1) >> 1, ey = 1 - (Y & 1), ex = 1 - (X & 1);
        int rowi[3][3];
#pragma unroll
        for (int i = 0; i < 3; ++i)
#pragma unroll
            for (int j = 0; j < 3; ++j) {
                const int64_t pi = pix0 + (int64_t)min(max(m0 + i, 0), h) * (w + 1) + min(max(n0 + j, 0), w);
                rowi[i][j] = __ldg(base + pi) + __popc(__ldg(need + pi) & below);
            }
        float4 e[4][4];
#pragma unroll
        for (int p = 0; p < 4; ++p)
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int u = Y - 1 + p, v = X - 1 + q;
                const int ra = ey ? (ex ? rowi[(p + 1) >> 1][(q + 1) >> 1] : rowi[(p + 1) >> 1][q >> 1])
                                  : (ex ? rowi[p >> 1][(q + 1) >> 1] : rowi[p >> 1][q >> 1]);
                e[p][q] = make_float4(0.f, 0.f, 0.f, 0.f);
                if (u >= 0 && v >= 0) e[p][q] = ld4(tb + ((int64_t)ra * 4 + (u & 1) * 2 + (v & 1)) * cout);
            }
        float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int p = 0; p < 4; ++p)
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const float c = __ldg(fir + 15 - 4 * p - q);
                a.x = fmaf(c, e[p][q].x, a.x), a.y = fmaf(c, e[p][q].y, a.y), a.z = fmaf(c, e[p][q].z, a.z), a.w = fmaf(c, e[p][q].w, a.w);
            }
        const float4 d = demod ? ld4(demod + ((int64_t)b * ncls + r) * cout + o) : make_float4(1.f, 1.f, 1.f, 1.f);
        const float4 bv = bias ? ld4(bias + o) : make_float4(0.f, 0.f, 0.f, 0.f);
        const float z = noise ? __ldg(noise_w) * __ldg(noise + ((int64_t)(noise_b == 1 ? 0 : b) * Ho + Y) * Wo + X) : 0.f;
        *reinterpret_cast<float4*>(y + (((int64_t)b * Ho + Y) * Wo + X) * cout + o) = epilogue4(a, d, z, bv, act);
    }
}

}  // namespace wgmma_conv

extern "C" int e4s_modconv3x3_up_tcr_fwd(const float* x, const void* wt_hilo_bf16, const float* fir4x4, const float* s,
                                         const float* demod, const float* noise, const float* noise_w, const float* bias,
                                         float* t_buf, float* y, int batch, int h, int w, int cin, int cout, int noise_b,
                                         int act, void* stream) {
    namespace wc = wgmma_conv;
    E4S_REQUIRE(fir4x4 && t_buf, E4S_ERR_ARG);
    if (const int rc = wc::check_modconv_fwd(x, wt_hilo_bf16, s, demod, nullptr, noise, noise_w, bias, y, batch, h, w, cin,
                                             cout, 1, noise_b, true))
        return rc;
    E4S_REQUIRE(e4s_aligned16(t_buf), E4S_ERR_ALIGN);
    cudaStream_t st = (cudaStream_t)stream;
    wc::Params p{};
    p.a = x, p.wt = static_cast<const __nv_bfloat16*>(wt_hilo_bf16), p.s = s, p.out = t_buf;
    p.batch = batch, p.h = h, p.w = w, p.mh = h + 1, p.mw = w + 1, p.kch = cin, p.nch = 4 * cout, p.ncls = 1;
    wc::tiles(p);
    if (const int rc = wc::launch_convt(p, (int64_t)p.tiles_x * p.tiles_y * batch * (cout / 32), st)) return rc;
    const int strips = (int)e4s_ceil_div(2 * h, wc::BLUR_ROWS);
    const int64_t blocks = e4s_ceil_div((int64_t)batch * strips * w * (cout / 4), wc::BLUR_THREADS);
    E4S_REQUIRE(blocks < (1ll << 31), E4S_ERR_SHAPE);
    wc::convt_blur_kernel<<<(unsigned)blocks, wc::BLUR_THREADS, 0, st>>>(t_buf, fir4x4, demod, noise, noise_w, bias, y, batch, h,
                                                                         w, cout, noise_b, act ? 1 : 0, strips);
    return e4s_launch_status();
}

extern "C" int e4s_modconv3x3_up_masked_tcr_fwd(const float* x, const void* wt_hilo_bf16, const void* w_hilo_bf16,
                                                const float* fir4x4, const float* s, const float* demod, const uint8_t* label,
                                                const float* noise, const float* noise_w, const float* bias, uint32_t* need,
                                                int* base, int* count, uint32_t* rows, float* t_buf, float* y, int batch, int h,
                                                int w, int cin, int cout, int ncls, int cap, int noise_b, int act, void* stream) {
    namespace wc = wgmma_conv;
    E4S_REQUIRE(w_hilo_bf16 && fir4x4 && label && need && base && count && rows && t_buf && cap > 0, E4S_ERR_ARG);
    if (const int rc = wc::check_modconv_fwd(x, wt_hilo_bf16, s, demod, label, noise, noise_w, bias, y, batch, h, w, cin,
                                             cout, ncls, noise_b, h + 1 < (1 << 14) && w + 1 < (1 << wc::ROW_NBITS)))
        return rc;
    E4S_REQUIRE(e4s_aligned16(w_hilo_bf16) && e4s_aligned16(t_buf), E4S_ERR_ALIGN);
    cudaStream_t st = (cudaStream_t)stream;
    wc::convt_row_list_kernel<<<batch, wc::LIST_THREADS, 0, st>>>(label, need, base, count, rows, h, w, ncls, cap);
    if (const int rc = e4s_launch_status()) return rc;
    // GEMM over each sample's rows in blocks of 128; blocks past the list's end cost one load
    wc::Params p{};
    p.a = x, p.wt = static_cast<const __nv_bfloat16*>(wt_hilo_bf16), p.s = s, p.out = t_buf, p.rows = rows, p.row_count = count;
    p.batch = batch, p.h = h, p.w = w, p.kch = cin, p.nch = 4 * cout, p.ncls = ncls, p.cap = cap;
    p.tiles_x = (int)e4s_ceil_div(cap, wc::M);
    const int nt = wc::pick_ntile_rows(cout, (int64_t)p.tiles_x * batch);
    if (const int rc = nt == 128 ? wc::launch_rows<128>(p, st) : nt == 64 ? wc::launch_rows<64>(p, st) : wc::launch_rows<32>(p, st))
        return rc;
    const int64_t blocks = e4s_ceil_div((int64_t)batch * 2 * h * e4s_ceil_div(2 * w, wc::BLUR_PIX) * (cout / 4), wc::BLUR_THREADS);
    E4S_REQUIRE(blocks < (1ll << 31), E4S_ERR_SHAPE);
    wc::convt_blur_masked_kernel<<<(unsigned)blocks, wc::BLUR_THREADS, 0, st>>>(t_buf, need, base, count, label, fir4x4, demod, noise,
                                                                                noise_w, bias, y, batch, h, w, cout, ncls, cap,
                                                                                noise_b, act ? 1 : 0);
    if (const int rc = e4s_launch_status()) return rc;
    // samples whose list overflowed: the folded parity kernel (its items for the other samples return at once)
    wc::Params f{};
    f.a = x, f.wt = static_cast<const __nv_bfloat16*>(w_hilo_bf16), f.s = s, f.demod = demod, f.label = label, f.row_count = count;
    f.noise = noise, f.noise_w = noise_w, f.bias = bias, f.out = y, f.cap = cap;
    f.batch = batch, f.h = h, f.w = w, f.kch = cin, f.nch = cout, f.ncls = ncls, f.noise_b = noise_b, f.act = act ? 1 : 0;
    f.up = 1;
    wc::set_taps(f, 0);
    return wc::forward(f, st);
}
