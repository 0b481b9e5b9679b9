// conv3x3_wgmma_kernel: the tensor-core 3x3 convolution with both operands staged in shared memory - the folded
// up-sampling forward (four output-parity convolutions on the input grid; the masked up-sampling layers' fallback for
// samples whose row list overflowed), the encoder's convolution, the BiSeNet bias convolution and the input / style
// gradient of the modulated convolution.  A work item is an 8 x 16 pixel tile
// (M = 128 rows) times an N tile of 32 or 64 output channels (one output parity of an up-sampling layer, or all four in
// turn); K runs over (parity plane, tap, 32-channel chunk).  Per K step the 256 threads stage
//   A: the 128 x 32 operand tile read from global memory at the tap's offset and scaled while staging - by the style of
//      each row's own output pixel (forward: every row may belong to another region, so a tile mixing regions needs no
//      extra pass), or by act'(y) * demod of the region whose pass it is (gradient: rows of other regions are zero);
//   B: the N x 32 weight tile from the pre-split bf16 planes,
// both as bf16 hi / lo planes (x = hi + lo to ~2^-17) in the no-swizzle K-major core-matrix layout of wgmma.  The two
// warpgroups (64 rows each) issue asynchronous wgmma.mma_async m64nNk16 with both operands from shared memory into
// fp32 register accumulators (split_mma).  The operand tiles go through a four-stage shared-memory ring: while the MMAs
// of step k run, the threads store step k + 2 (loaded from global memory one step earlier) and issue the loads of step
// k + 3; one barrier per K step.  The operands cannot be copied by TMA: every element is scaled and split on its way
// into shared memory.  Every output element is accumulated in a fixed order, so the forward is bit reproducible; the
// gradient sums split work items and style gradients with atomics.
#include "wgmma_conv.cuh"

namespace wgmma_conv {

__device__ __forceinline__ uint32_t pack2(__nv_bfloat16 lo_elem, __nv_bfloat16 hi_elem) {
    return (uint32_t)__bfloat16_as_ushort(lo_elem) | ((uint32_t)__bfloat16_as_ushort(hi_elem) << 16);
}
// four fp32 values -> bf16 hi plane and residual lo plane, 8 bytes each
__device__ __forceinline__ void split_store4(float4 v, __nv_bfloat16* hi, __nv_bfloat16* lo) {
    const __nv_bfloat16 h0 = __float2bfloat16_rn(v.x), h1 = __float2bfloat16_rn(v.y), h2 = __float2bfloat16_rn(v.z),
                        h3 = __float2bfloat16_rn(v.w);
    const __nv_bfloat16 l0 = __float2bfloat16_rn(v.x - __bfloat162float(h0)), l1 = __float2bfloat16_rn(v.y - __bfloat162float(h1)),
                        l2 = __float2bfloat16_rn(v.z - __bfloat162float(h2)), l3 = __float2bfloat16_rn(v.w - __bfloat162float(h3));
    *reinterpret_cast<uint2*>(hi) = make_uint2(pack2(h0, h1), pack2(h2, h3));
    *reinterpret_cast<uint2*>(lo) = make_uint2(pack2(l0, l1), pack2(l2, l3));
}
__device__ __forceinline__ float4 mul4(float4 a, float4 b) { return make_float4(a.x * b.x, a.y * b.y, a.z * b.z, a.w * b.w); }
__device__ __forceinline__ float actd(float y) { return y > 0.f ? SQRT2 : 0.2f * SQRT2; }

// FWD_BIAS: o = acc + bias[n] + residual, then ReLU when p.act; res points at the residual element of dst (or NULL)
__device__ __forceinline__ void epilogue_bias2(const Params& p, int n, float a0, float a1, const float* res, float* dst) {
    float2 o = make_float2(a0, a1);
    if (p.bias) {
        const float2 bv = __ldg(reinterpret_cast<const float2*>(p.bias + n));
        o.x += bv.x, o.y += bv.y;
    }
    if (res) {
        const float2 rv = *reinterpret_cast<const float2*>(res + n);
        o.x += rv.x, o.y += rv.y;
    }
    if (p.act) o.x = fmaxf(o.x, 0.f), o.y = fmaxf(o.y, 0.f);
    *reinterpret_cast<float2*>(dst + n) = o;
}

template <int NT, int MODE>
__global__ void __launch_bounds__(NUM_THREADS, (MODE == BWD || NT == 32) ? 1 : 2) conv3x3_wgmma_kernel(const Params p) {
    constexpr bool GRAD = MODE == BWD;
    static_assert(NT == 32 || NT == 64, "N tiles of 32 or 64");
    constexpr int NR = NT / 2;                        // accumulator registers per thread (m64 x NT per warpgroup)
    constexpr int BVEC = NT * KC / 8;                 // 16-byte vectors per B plane and K step
    constexpr int BV = (BVEC + NUM_THREADS - 1) / NUM_THREADS;
    constexpr int B_PLANE = NT * KC * 2;
    constexpr int STAGE = 2 * A_PLANE + 2 * B_PLANE;  // [A hi | A lo | B hi | B lo]
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    __shared__ uint32_t s_classes;

    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const int wg = warp >> 2, wi = warp & 3;          // warpgroup (rows 64 wg ..), warp within it
    Item it = decode_item<true>(p, blockIdx.x, NT * p.n_sub);
    const int b = it.b, idx = it.rest;
    int n0 = it.n0;
    const int mul = p.up ? 2 : 1;
    const int H = p.h, W = p.w, MH = p.mh, MW = p.mw, Ho = MH * mul, Wo = MW * mul;
    const int y0 = it.ty * TH, x0 = it.tx * TW;
    if (!GRAD && p.row_count && __ldg(p.row_count + b) <= p.cap) return;    // masked fallback: overflowed samples only
    const int nphw = p.up ? 4 : 1;                    // parity planes of the weights
    // FWD: idx = output parity of the item.  BWD: idx = region-pass group + gsplit * parity-plane group.
    int par = GRAD ? 0 : idx;
    const int g = GRAD ? idx % p.gsplit : 0;
    const int ph0 = GRAD ? (idx / p.gsplit) * (nphw / p.hsplit) : 0;
    const int nph_k = GRAD ? nphw / p.hsplit : 1;
    int py = par >> 1, px = par & 1;
    const int c4 = t & 7, rr = t >> 3;                // A staging: channel group, first row
    const int nchunks = p.kch / KC;
    const int nsteps = nph_k * p.ntaps * nchunks;
    const int64_t plane = (int64_t)p.nch * p.kch;

    // forward: region of each staged row's own output pixel
    int rcls[4] = {0, 0, 0, 0};
    auto row_classes = [&]() {
        if (!p.label) return;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int r = rr + 32 * j, iy = y0 + (r >> 4), ix = x0 + (r & 15);
            if (iy < MH && ix < MW) rcls[j] = region(p.label, p.ncls, ((int64_t)b * Ho + iy * mul + py) * Wo + ix * mul + px);
        }
    };

    float4 av[4], am[4], ad;
    bool aok[4];
    uint4 bh[BV], bl[BV];
    auto load = [&](int step, int pass) {
        const int kc = step % nchunks;
        const int rest = step / nchunks;
        const int tap = p.taps[rest % p.ntaps];
        const int ph = ph0 + rest / p.ntaps;
        const int dy = tap / 3, dx = tap % 3;
        const int k = kc * KC + c4 * 4;
        if (GRAD) ad = p.demod ? ld4(p.demod + ((int64_t)b * p.ncls + pass) * p.kch + k) : make_float4(1.f, 1.f, 1.f, 1.f);
        else ad = p.shift ? ld4(p.shift + (int64_t)b * p.kch + k) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int r = rr + 32 * j;
            const int iy = y0 + (r >> 4), ix = x0 + (r & 15);
            const int sy = iy + dy - 1, sx = ix + dx - 1;
            bool ok = iy < MH && ix < MW && sy >= 0 && sy < H && sx >= 0 && sx < W;
            av[j] = make_float4(0.f, 0.f, 0.f, 0.f);
            am[j] = make_float4(1.f, 1.f, 1.f, 1.f);
            if (GRAD) {
                const int64_t gp = ((int64_t)b * Ho + sy * mul + (ph >> 1)) * Wo + sx * mul + (ph & 1);
                if (ok && p.label) ok = region(p.label, p.ncls, gp) == pass;
                if (ok) {
                    av[j] = ld4(p.a + gp * p.kch + k);
                    if (p.y) am[j] = ld4(p.y + gp * p.kch + k);
                }
            } else if (ok) {
                av[j] = ld4(p.a + (((int64_t)b * H + sy) * W + sx) * p.kch + k);
                if (p.s) am[j] = ld4(p.s + ((int64_t)b * p.ncls + rcls[j]) * p.kch + k);
            }
            aok[j] = ok;
        }
#pragma unroll
        for (int v = 0; v < BV; ++v) {                // B: 16-byte vectors of both planes
            const int e = t + NUM_THREADS * v;
            if (e < BVEC) {
                const int n = n0 + (e >> 2), kk = kc * KC + (e & 3) * 8;
                const int wph = GRAD ? ph : par;
                const int64_t off = (int64_t)(wph * 9 + tap) * plane + (int64_t)n * p.kch + kk;
                bh[v] = __ldg(reinterpret_cast<const uint4*>(p.wt + off));
                bl[v] = __ldg(reinterpret_cast<const uint4*>(p.wt + (int64_t)nphw * 9 * plane + off));
            }
        }
    };
    auto store = [&](int buf) {
        uint8_t* st = smem + buf * STAGE;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int r = rr + 32 * j;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (aok[j]) {
                if (GRAD) {
                    const float4 d = p.y ? make_float4(actd(am[j].x), actd(am[j].y), actd(am[j].z), actd(am[j].w)) : am[j];
                    v = mul4(mul4(av[j], d), ad);
                } else {
                    v = make_float4(av[j].x * am[j].x + ad.x, av[j].y * am[j].y + ad.y, av[j].z * am[j].z + ad.z,
                                    av[j].w * am[j].w + ad.w);
                }
            }
            const int off = (r >> 3) * SBO + (c4 >> 1) * LBO + (r & 7) * 16 + (c4 & 1) * 8;
            split_store4(v, reinterpret_cast<__nv_bfloat16*>(st + off), reinterpret_cast<__nv_bfloat16*>(st + A_PLANE + off));
        }
#pragma unroll
        for (int v = 0; v < BV; ++v) {
            const int e = t + NUM_THREADS * v;
            if (e < BVEC) {
                const int n = e >> 2;
                const int off = 2 * A_PLANE + (n >> 3) * SBO + (e & 3) * LBO + (n & 7) * 16;
                *reinterpret_cast<uint4*>(st + off) = bh[v];
                *reinterpret_cast<uint4*>(st + off + B_PLANE) = bl[v];
            }
        }
    };
    SplitAcc<NT> acc{};                               // zero: the fences read every register
    const uint32_t smem_s = (uint32_t)__cvta_generic_to_shared(smem);
    // the split-precision products of one K step, both K16 slices, on ring slot `buf`
    auto issue = [&](int buf, bool first) {
        const uint32_t a_hi = smem_s + buf * STAGE + wg * (64 / 8) * SBO, a_lo = a_hi + A_PLANE;
        const uint32_t b_hi = smem_s + buf * STAGE + 2 * A_PLANE, b_lo = b_hi + B_PLANE;
        acc.fence();
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < KC / 16; ++ks) {
            const uint32_t ko = ks * 2 * LBO;
            const int accumulate = (first && ks == 0) ? 0 : 1;
            split_mma(acc, a_hi + ko, a_lo + ko, b_hi + ko, b_lo + ko, accumulate);
        }
        wgmma_commit();
        acc.fence();
    };
    // Ring: slot k % NSTAGE holds step k.  Iteration k issues step k, waits until only it is in flight (so step k - 1 is
    // done in this warpgroup), stores step k + 2 into the slot of step k - 2 (done in both warpgroups: the barrier of
    // iteration k - 1 followed their waits), loads step k + 3 into registers, and meets the other threads at the barrier.
    // (the first MMA of a pass overwrites the accumulators: no register write may sit between asynchronous MMAs)
    auto run = [&](int pass) {
        load(0, pass);
        store(0);
        if (1 < nsteps) load(1, pass), store(1);
        if (2 < nsteps) load(2, pass);
        fence_proxy_async();
        __syncthreads();
#pragma unroll 1
        for (int st = 0; st < nsteps; ++st) {
            issue(st % NSTAGE, st == 0);
            wgmma_wait<1>();
            acc.fence();
            if (st + 2 < nsteps) store((st + 2) % NSTAGE);
            if (st + 3 < nsteps) load(st + 3, pass);
            fence_proxy_async();
            __syncthreads();
        }
        wgmma_wait<0>();
        acc.fence();
        __syncthreads();                              // every slot free before a following pass stores into it
        acc.fold();
    };
    auto row_of = [&](int hf) { return wg * 64 + wi * 16 + (lane >> 2) + 8 * hf; };
    auto col_of = [&](int j) { return n0 + j * 8 + 2 * (lane & 3); };

    if (!GRAD) {
        // one output parity per item, or (up-sampling layer, parity_items == 0) all four in turn
        const bool all4 = p.up && !p.parity_items;
#pragma unroll 1
        for (int q = all4 ? 0 : par; q < (all4 ? 4 : par + 1); ++q) {
            par = q, py = q >> 1, px = q & 1;
            row_classes();
            run(0);
            const float nw = (p.noise && p.noise_w) ? __ldg(p.noise_w) : 0.f;
            const bool strided = p.out_stride != 1;
            const int oh = strided ? H / 2 : Ho, ow = strided ? W / 2 : Wo;
#pragma unroll
            for (int hf = 0; hf < 2; ++hf) {
                    const int r = row_of(hf), iy = y0 + (r >> 4), ix = x0 + (r & 15);
                    if (iy >= MH || ix >= MW || (p.out_stride == 2 && ((iy | ix) & 1))) continue;
                    const int oy = iy * mul + py, ox = ix * mul + px;
                    const int cls = p.label ? region(p.label, p.ncls, ((int64_t)b * Ho + oy) * Wo + ox) : 0;
                    const float z = p.noise ? nw * __ldg(p.noise + ((int64_t)(p.noise_b == 1 ? 0 : b) * Ho + oy) * Wo + ox) : 0.f;
                    float* dst;
                    if (p.out_stride == 4)
                        dst = p.out + (((int64_t)b * oh + (iy >> 1)) * ow + (ix >> 1)) * 4 * p.nch + ((iy & 1) * 2 + (ix & 1)) * p.nch;
                    else if (strided)
                        dst = p.out + (((int64_t)b * oh + (iy >> 1)) * ow + (ix >> 1)) * p.nch;
                    else
                        dst = p.out + (((int64_t)b * Ho + oy) * Wo + ox) * p.nch;
                    if constexpr (MODE == FWD_BIAS) {
                        const float* res = p.residual ? p.residual + (dst - p.out) : nullptr;
#pragma unroll
                        for (int nf = 0; nf < NT / 8; ++nf)
                            epilogue_bias2(p, col_of(nf), acc.d[4 * nf + 2 * hf], acc.d[4 * nf + 2 * hf + 1], res, dst);
                    } else {
#pragma unroll
                        for (int nf = 0; nf < NT / 8; ++nf)
                            epilogue2<true>(p, b, cls, col_of(nf), z, acc.d[4 * nf + 2 * hf], acc.d[4 * nf + 2 * hf + 1], dst);
                    }
                }
        }
        return;
    }

    // ---- gradient: one pass per region present among the tile's source pixels (this item's share of them)
    uint32_t classes = 1u;
    if (p.label) {
        if (t == 0) s_classes = 0u;
        __syncthreads();
        uint32_t m = 0;
        const int nhalo = (TH + 2) * (TW + 2);
        for (int e = t; e < nhalo * nph_k; e += NUM_THREADS) {
            const int hp = e % nhalo, ph = ph0 + e / nhalo;
            const int sy = y0 - 1 + hp / (TW + 2), sx = x0 - 1 + hp % (TW + 2);
            if (sy >= 0 && sy < H && sx >= 0 && sx < W)
                m |= 1u << region(p.label, p.ncls, ((int64_t)b * Ho + sy * mul + (ph >> 1)) * Wo + sx * mul + (ph & 1));
        }
        m = __reduce_or_sync(0xffffffffu, m);
        if (lane == 0 && m) atomicOr(&s_classes, m);
        __syncthreads();
        classes = s_classes;
    }
#pragma unroll 1
    for (int sub = 0; sub < p.n_sub; ++sub) {           // N tiles of this work item
    n0 = it.n0 + sub * NT;
        float gxa[NR];
#pragma unroll
        for (int i = 0; i < NR; ++i) gxa[i] = 0.f;
        int k = 0;
        for (uint32_t cm = classes; cm; cm &= cm - 1, ++k) {
            if (k % p.gsplit != g) continue;
            const int c = __ffs(cm) - 1;
            run(c);
            const float* sc = p.s + ((int64_t)b * p.ncls + c) * p.nch;
#pragma unroll
            for (int nf = 0; nf < NT / 8; ++nf) {
                const int n = col_of(nf);
                const float2 s2 = __ldg(reinterpret_cast<const float2*>(sc + n));
                float gs0 = 0.f, gs1 = 0.f;
#pragma unroll
                for (int hf = 0; hf < 2; ++hf) {
                        const float u0 = acc.d[4 * nf + 2 * hf], u1 = acc.d[4 * nf + 2 * hf + 1];
                        gxa[4 * nf + 2 * hf] += s2.x * u0, gxa[4 * nf + 2 * hf + 1] += s2.y * u1;
                        if (p.gs) {
                            const int r = row_of(hf), iy = y0 + (r >> 4), ix = x0 + (r & 15);
                            if (iy < H && ix < W) {
                                const float2 xv = __ldg(reinterpret_cast<const float2*>(p.x + (((int64_t)b * H + iy) * W + ix) * p.nch + n));
                                gs0 += xv.x * u0, gs1 += xv.y * u1;
                            }
                        }
                    }
                if (p.gs) {
#pragma unroll
                    for (int o = 4; o < 32; o <<= 1) gs0 += __shfl_xor_sync(0xffffffffu, gs0, o), gs1 += __shfl_xor_sync(0xffffffffu, gs1, o);
                    if (lane < 4) {
                        float* gp = p.gs + ((int64_t)b * p.ncls + c) * p.nch + n;
                        atomicAdd(gp, gs0);
                        atomicAdd(gp + 1, gs1);
                    }
                }
            }
        }
        if (!p.out) continue;
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
                const int r = row_of(hf), iy = y0 + (r >> 4), ix = x0 + (r & 15);
                if (iy >= H || ix >= W) continue;
                float* dst = p.out + (((int64_t)b * H + iy) * W + ix) * p.nch;
#pragma unroll
                for (int nf = 0; nf < NT / 8; ++nf) {
                    const int n = col_of(nf);
                    if (p.atomic_gx) {
                        atomicAdd(dst + n, gxa[4 * nf + 2 * hf]);
                        atomicAdd(dst + n + 1, gxa[4 * nf + 2 * hf + 1]);
                    } else {
                        *reinterpret_cast<float2*>(dst + n) = make_float2(gxa[4 * nf + 2 * hf], gxa[4 * nf + 2 * hf + 1]);
                    }
                }
            }
    }
}

// ------------------------------------------------------------------------------------------ host
// Gradient work items: a (pixel tile, N tile) pair is a serial chain of (regions in the tile) x parity planes x taps x
// Cout / 32 K steps.  The low-resolution layers of one face have a handful of pairs with every region in each: when the
// pairs cannot fill the SMs, cut the chain - region passes first (up to ncls ways), then parity planes; the partial sums
// meet in gx through atomics (gx zeroed first) and in gs through the atomics the kernel uses anyway.
// E4S_B200_DGRAD_SPLIT="G,H" forces a split (tests).
static void choose_split(int64_t pairs, int ncls, int nph, int& gsplit, int& hsplit) {
    gsplit = hsplit = 1;
    if (const char* f = getenv("E4S_B200_DGRAD_SPLIT")) {
        int g = 0, h = 0;
        if (sscanf(f, "%d,%d", &g, &h) == 2 && g >= 1 && (h == 1 || h == 2 || h == 4)) {
            gsplit = g < ncls ? g : ncls, hsplit = h < nph ? h : nph;
            return;
        }
    }
    const int sms = num_sms();
    if (pairs >= 2 * sms) return;
    // aim at ~4 work items per SM: the chains differ in length (regions per tile)
    const int64_t g = e4s_ceil_div(4 * sms, pairs);
    gsplit = (int)(g < ncls ? g : ncls);
    while (hsplit < nph && pairs * gsplit * hsplit < sms) hsplit *= 2;
}

template <int NT, int MODE>
static int launch_smem(Params p, int64_t outer, cudaStream_t st) {
    p.n_tiles = p.nch / NT;
    const int64_t items = (int64_t)p.tiles_x * p.tiles_y * p.batch * p.n_tiles * outer;
    if (items >= (1ll << 31)) return E4S_ERR_SHAPE;
    constexpr size_t smem = 1024 + (size_t)NSTAGE * (2 * A_PLANE + 2 * NT * KC * 2);
    static E4sSmemOptIn optin;
    if (const int rc = e4s_smem_optin(optin, conv3x3_wgmma_kernel<NT, MODE>, smem)) return rc;
    conv3x3_wgmma_kernel<NT, MODE><<<(unsigned)items, NUM_THREADS, smem, st>>>(p);
    return e4s_launch_status();
}

// nt: channels per work item (pick_ntile)
template <int MODE>
static int launch(const Params& p, int nt, int64_t outer, cudaStream_t st) {
    return nt == 32 ? launch_smem<32, MODE>(p, outer, st) : launch_smem<64, MODE>(p, outer, st);
}

template <int MODE>
int forward(Params p, cudaStream_t st) {
    tiles(p);
    const int64_t pixel_tiles = (int64_t)p.tiles_x * p.tiles_y * p.batch;
    // up-sampling layer: one output parity per work item, or all four in one item once the items already fill the GPU
    // twice over without the split (four times fewer operand-ring fills); E4S_B200_UP2=1 | 0 forces either (tests)
    const int nt = pick_ntile(p.nch, pixel_tiles * (p.up ? 4 : 1));
    p.parity_items = pixel_tiles * (p.nch / nt) < 2 * num_sms();
    if (const char* f = getenv("E4S_B200_UP2")) p.parity_items = atoi(f) != 0;
    const int64_t outer = (p.up && p.parity_items) ? 4 : 1;
    return launch<MODE>(p, nt, outer, st);
}
template int forward<FWD>(Params p, cudaStream_t st);

}  // namespace wgmma_conv

// Arguments common to the two plain-convolution entry points into p; the first failing check gives the error code.
// `extra` is every further pointer of the entry (each may be NULL), checked for 16-byte alignment.
static int plain_conv_params(wgmma_conv::Params& p, const float* x, const void* w_hilo_bf16, const float* scale,
                             const float* shift, float* y, int batch, int h, int w, int cin, int cout, int out_stride,
                             int tap_mask, std::initializer_list<const void*> extra) {
    E4S_REQUIRE(x && w_hilo_bf16 && y, E4S_ERR_ARG);
    E4S_REQUIRE(tap_mask >= 0 && tap_mask <= 0x1FF, E4S_ERR_ARG);
    E4S_REQUIRE(batch > 0 && h > 0 && w > 0 && cin > 0 && cout > 0, E4S_ERR_ARG);
    E4S_REQUIRE((cin % 32) == 0 && (cout % 32) == 0, E4S_ERR_SHAPE);
    E4S_REQUIRE(out_stride == 1 || ((out_stride == 2 || out_stride == 4) && (h % 2) == 0 && (w % 2) == 0), E4S_ERR_SHAPE);
    E4S_REQUIRE(e4s_aligned16(x) && e4s_aligned16(w_hilo_bf16) && e4s_aligned16(y) && (!scale || e4s_aligned16(scale)) &&
                    (!shift || e4s_aligned16(shift)),
                E4S_ERR_ALIGN);
    for (const void* q : extra) E4S_REQUIRE(!q || e4s_aligned16(q), E4S_ERR_ALIGN);
    p.a = x, p.wt = static_cast<const __nv_bfloat16*>(w_hilo_bf16), p.s = scale, p.shift = shift, p.out = y;
    p.batch = batch, p.h = h, p.w = w, p.kch = cin, p.nch = cout, p.ncls = 1;
    p.out_stride = out_stride;
    wgmma_conv::set_taps(p, tap_mask);
    return E4S_OK;
}

extern "C" int e4s_conv3x3_tcr_f32(const float* x, const void* w_hilo_bf16, const float* scale, const float* shift,
                                   const float* prelu_slope, float* y, int batch, int h, int w, int cin, int cout,
                                   int out_stride, int tap_mask, void* stream) {
    wgmma_conv::Params p{};
    if (const int rc = plain_conv_params(p, x, w_hilo_bf16, scale, shift, y, batch, h, w, cin, cout, out_stride, tap_mask,
                                         {prelu_slope}))
        return rc;
    p.slope = prelu_slope, p.act = prelu_slope ? 2 : 0;
    return wgmma_conv::forward(p, (cudaStream_t)stream);
}

extern "C" int e4s_conv3x3_bias_tcr_f32(const float* x, const void* w_hilo_bf16, const float* scale, const float* shift,
                                        const float* bias, const float* residual, float* y, int batch, int h, int w, int cin,
                                        int cout, int out_stride, int tap_mask, int relu, void* stream) {
    wgmma_conv::Params p{};
    if (const int rc = plain_conv_params(p, x, w_hilo_bf16, scale, shift, y, batch, h, w, cin, cout, out_stride, tap_mask,
                                         {bias, residual}))
        return rc;
    p.bias = bias, p.residual = residual, p.act = relu ? 1 : 0;
    return wgmma_conv::forward<wgmma_conv::FWD_BIAS>(p, (cudaStream_t)stream);
}

extern "C" int e4s_modconv3x3_bwd_tc(const float* gy, const float* y, const float* x, const void* wd_hilo_bf16, const float* s,
                                     const float* demod, const uint8_t* label, float* gx, float* gs, int batch, int h, int w,
                                     int cin, int cout, int ncls, int up, int act, void* stream) {
    E4S_REQUIRE(gy && wd_hilo_bf16 && s && (gx || gs), E4S_ERR_ARG);
    E4S_REQUIRE(!act || y, E4S_ERR_ARG);
    E4S_REQUIRE(!gs || x, E4S_ERR_ARG);
    E4S_REQUIRE(batch > 0 && h > 0 && w > 0 && cin > 0 && cout > 0 && ncls > 0 && ncls <= 32, E4S_ERR_ARG);
    E4S_REQUIRE((cin % 32) == 0 && (cout % 32) == 0, E4S_ERR_SHAPE);
    E4S_REQUIRE(label || ncls == 1, E4S_ERR_ARG);
    cudaStream_t st = (cudaStream_t)stream;
    wgmma_conv::Params p{};
    p.a = gy, p.y = act ? y : nullptr, p.x = x, p.wt = static_cast<const __nv_bfloat16*>(wd_hilo_bf16), p.s = s, p.demod = demod;
    p.label = label, p.out = gx, p.gs = gs;
    p.batch = batch, p.h = h, p.w = w, p.kch = cout, p.nch = cin, p.ncls = ncls, p.act = act ? 1 : 0;
    p.up = up ? 1 : 0;
    wgmma_conv::set_taps(p, 0);
    wgmma_conv::tiles(p);
    const int nph = up ? 4 : 1;
    const int64_t pixel_tiles = (int64_t)p.tiles_x * p.tiles_y * batch;
    const int nt = wgmma_conv::pick_ntile(cin, pixel_tiles);
    wgmma_conv::choose_split(pixel_tiles * (cin / nt), label ? ncls : 1, nph, p.gsplit, p.hsplit);
    p.atomic_gx = p.gsplit * p.hsplit > 1;
    if (p.atomic_gx && gx && cudaMemsetAsync(gx, 0, (size_t)batch * h * w * cin * sizeof(float), st) != cudaSuccess)
        return (int)cudaGetLastError();
    return wgmma_conv::launch<wgmma_conv::BWD>(p, nt, (int64_t)p.gsplit * p.hsplit, st);
}

// Host-only: the work list e4s_modconv3x3_bwd_tc builds for this shape (N-tile width, region-pass and parity-plane split).
// ncls = number of regions the label map can hold (1 without one).  No launch, no device access beyond the SM count
// (132 when no device is present) - lets the host-side heuristics be tested without a GPU.
extern "C" int e4s_modconv3x3_bwd_tc_plan(int batch, int h, int w, int cin, int ncls, int up, int* ntile, int* gsplit, int* hsplit) {
    E4S_REQUIRE(ntile && gsplit && hsplit && batch > 0 && h > 0 && w > 0 && cin > 0 && ncls > 0 && ncls <= 32, E4S_ERR_ARG);
    E4S_REQUIRE((cin % 32) == 0, E4S_ERR_SHAPE);
    const int64_t pixel_tiles = e4s_ceil_div(w, wgmma_conv::TW) * e4s_ceil_div(h, wgmma_conv::TH) * batch;
    *ntile = wgmma_conv::pick_ntile(cin, pixel_tiles);
    wgmma_conv::choose_split(pixel_tiles * (cin / *ntile), ncls, up ? 4 : 1, *gsplit, *hsplit);
    return E4S_OK;
}
