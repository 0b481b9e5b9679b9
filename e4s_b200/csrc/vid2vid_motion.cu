// The passes of face-vid2vid's dense-motion network (src/pretrained/face_vid2vid/modules/dense_motion.py,
// DenseMotionNetwork on vox-256.yaml) around its tensor-core convolutions:
//   * compress: the 1x1x1 convolution 32 -> 4 with its BatchNorm folded in, then ReLU, from the NCDHW feature to one
//     float4 per voxel [B, D, H, W, 4], so that a trilinear corner is one 16-byte load;
//   * the hourglass input: per voxel the 16 trilinear samples of the compressed volume at the sparse motions (the
//     identity grid, then grid - kp_driving[k] + kp_source[k]; F.grid_sample's defaults: align_corners=False, zero
//     padding) and the 15 heatmap differences, as channel 5 k + j (j = 0 the heatmap, 1..4 the sample), 80 channels and
//     16 zeros, into a channel slice of the hourglass's [B, H, W, D, *] level-0 buffer;
//   * AvgPool3d((1, 2, 2)) of a [B, H, W, D, C] volume into a channel slice of a wider buffer;
//   * the mask / occlusion combine after the per-slice 7x7 GEMM (e4s_conv7x7_slices_tcr_f32): the 7x7x7 mask logits as
//     sums of the GEMM's (dz, o) columns over the depths, the 16-way softmax, the deformation and the occlusion map;
//   * the SPADE generator's deform_input: the trilinear samples of its 32-channel [B, H, W, D, 32] feature volume at the
//     deformation, written as the [B, H, W, D 32] operand of its `third` convolution (the same sampler as the hourglass
//     input).
// Every sum runs in a fixed order that depends on neither the batch nor the launch: bit reproducible, batch-invariant.
#include "common.cuh"

namespace v2vdm {

constexpr int THREADS = 256;
constexpr int NKP = 15, NK = NKP + 1, CC = 4, CF = 32;     // keypoints, sparse motions, compressed / feature channels
constexpr int IN_CH = NK * (CC + 1), IN_PAD = 96;          // hourglass input channels, zero-padded
constexpr int MASK_TAPS = 7, OCC_COL = MASK_TAPS * NK;     // GEMM columns: (dz, o) mask weights, then occlusion per depth
constexpr int P_COLS = 128;

// make_coordinate_grid: 2 (i / (n - 1)) - 1, in fp32 as the reference computes it
__device__ __forceinline__ float coord(int i, int n) { return 2.f * ((float)i / (float)(n - 1)) - 1.f; }

// one thread per voxel v of sample b: y[b, v, j] = relu(bias[j] + sum over c of w[j, c] x[b, c, v]), c in order
__global__ void __launch_bounds__(THREADS) compress_kernel(const float* __restrict__ x, const float* __restrict__ wb,
                                                           float* __restrict__ y, int nvox) {
    __shared__ float sw[CC * CF + CC];
    for (int e = threadIdx.x; e < CC * CF + CC; e += THREADS) sw[e] = __ldg(wb + e);
    __syncthreads();
    const int v = blockIdx.x * THREADS + threadIdx.x, b = blockIdx.y;
    if (v >= nvox) return;
    const float* xb = x + (int64_t)b * CF * nvox + v;
    float a[CC] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 8
    for (int c = 0; c < CF; ++c) {
        const float xv = __ldg(xb + (int64_t)c * nvox);
#pragma unroll
        for (int j = 0; j < CC; ++j) a[j] = fmaf(sw[j * CF + c], xv, a[j]);
    }
    reinterpret_cast<float4*>(y)[(int64_t)b * nvox + v] =
        make_float4(fmaxf(a[0] + sw[CC * CF], 0.f), fmaxf(a[1] + sw[CC * CF + 1], 0.f), fmaxf(a[2] + sw[CC * CF + 2], 0.f),
                    fmaxf(a[3] + sw[CC * CF + 3], 0.f));
}

// F.grid_sample (trilinear, zero padding, align_corners=False) of a float4 volume of depth d, height h and width w at the
// normalised point (gx, gy, gz), voxel (z, y, x) at vol[z sz + y sy + x sx]: the eight corners in torch's order (tnw, tne,
// tsw, tse, bnw, bne, bsw, bse), out-of-volume corners skipped
__device__ __forceinline__ float4 sample(const float4* __restrict__ vol, int64_t sz, int64_t sy, int64_t sx, float gx, float gy,
                                         float gz, int d, int h, int w) {
    const float ix = ((gx + 1.f) * w - 1.f) / 2.f, iy = ((gy + 1.f) * h - 1.f) / 2.f, iz = ((gz + 1.f) * d - 1.f) / 2.f;
    const float fx = floorf(ix), fy = floorf(iy), fz = floorf(iz);
    const int x0 = (int)fx, y0 = (int)fy, z0 = (int)fz;
    const float wx[2] = {(fx + 1.f) - ix, ix - fx}, wy[2] = {(fy + 1.f) - iy, iy - fy}, wz[2] = {(fz + 1.f) - iz, iz - fz};
    float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int c = 0; c < 8; ++c) {
        const int cz = c >> 2, cy = (c >> 1) & 1, cx = c & 1;
        const int xx = x0 + cx, yy = y0 + cy, zz = z0 + cz;
        if (xx < 0 || xx >= w || yy < 0 || yy >= h || zz < 0 || zz >= d) continue;
        const float wt = wx[cx] * wy[cy] * wz[cz];
        const float4 v = __ldg(vol + zz * sz + yy * sy + xx * sx);
        o.x = fmaf(wt, v.x, o.x), o.y = fmaf(wt, v.y, o.y), o.z = fmaf(wt, v.z, o.z), o.w = fmaf(wt, v.w, o.w);
    }
    return o;
}

// one thread per output voxel (b, z, y, x) (x fastest): its 96 hourglass input channels at y_out + voxel * vp
__global__ void __launch_bounds__(THREADS) motion_input_kernel(const float4* __restrict__ comp, const float* __restrict__ kd,
                                                               const float* __restrict__ ks, float* __restrict__ out, int vp,
                                                               int d, int h, int w) {
    const int hw = h * w, i = blockIdx.x * THREADS + threadIdx.x, z = blockIdx.y, b = blockIdx.z;
    if (i >= hw) return;
    const int y = i / w, x = i - y * w;
    const float gx = coord(x, w), gy = coord(y, h), gz = coord(z, d);
    const float4* vol = comp + (int64_t)b * d * hw;
    const float* kdb = kd + b * NKP * 3;
    const float* ksb = ks + b * NKP * 3;
    float ch[IN_PAD];
#pragma unroll
    for (int k = 0; k < NK; ++k) {
        float mx = gx, my = gy, mz = gz, hm = 0.f;
        if (k > 0) {
            const float dx = __ldg(kdb + 3 * (k - 1)), dy = __ldg(kdb + 3 * (k - 1) + 1), dz = __ldg(kdb + 3 * (k - 1) + 2);
            const float sx = __ldg(ksb + 3 * (k - 1)), sy = __ldg(ksb + 3 * (k - 1) + 1), sz = __ldg(ksb + 3 * (k - 1) + 2);
            mx = (gx - dx) + sx, my = (gy - dy) + sy, mz = (gz - dz) + sz;
            const float ed = (gx - dx) * (gx - dx) + (gy - dy) * (gy - dy) + (gz - dz) * (gz - dz);
            const float es = (gx - sx) * (gx - sx) + (gy - sy) * (gy - sy) + (gz - sz) * (gz - sz);
            hm = expf(-0.5f * ed / 0.01f) - expf(-0.5f * es / 0.01f);
        }
        const float4 v = sample(vol, hw, w, 1, mx, my, mz, d, h, w);
        ch[5 * k] = hm, ch[5 * k + 1] = v.x, ch[5 * k + 2] = v.y, ch[5 * k + 3] = v.z, ch[5 * k + 4] = v.w;
    }
#pragma unroll
    for (int c = IN_CH; c < IN_PAD; ++c) ch[c] = 0.f;
    float4* dst = reinterpret_cast<float4*>(out + ((((int64_t)b * h + y) * w + x) * d + z) * vp);
#pragma unroll
    for (int c = 0; c < IN_PAD / 4; ++c) dst[c] = make_float4(ch[4 * c], ch[4 * c + 1], ch[4 * c + 2], ch[4 * c + 3]);
}

// [B, H, W, D, C] -> [B, H / 2, W / 2, D, C] at voxel pitch vp: (((x00 + x01) + x10) + x11) / 4, a float4 per thread
__global__ void __launch_bounds__(THREADS) avgpool2_vox_kernel(const float* __restrict__ x, float* __restrict__ y, int64_t total4,
                                                               int h, int w, int d, int c4, int vp) {
    const int64_t i = (int64_t)blockIdx.x * THREADS + threadIdx.x;
    if (i >= total4) return;
    const int ho = h >> 1, wo = w >> 1, dc4 = d * c4;
    const int e = (int)(i % dc4);
    int64_t r = i / dc4;
    const int ox = (int)(r % wo);
    r /= wo;
    const int oy = (int)(r % ho);
    const int64_t b = r / ho;
    const float4* s = reinterpret_cast<const float4*>(x) + ((b * h + 2 * oy) * w + 2 * ox) * dc4 + e;
    const float4 a = __ldg(s), bb = __ldg(s + dc4), c = __ldg(s + (int64_t)w * dc4), dd = __ldg(s + (int64_t)w * dc4 + dc4);
    const int z = e / c4, q = e - z * c4;
    reinterpret_cast<float4*>(y + (((b * ho + oy) * wo + ox) * d + z) * vp)[q] =
        make_float4((((a.x + bb.x) + c.x) + dd.x) / 4.f, (((a.y + bb.y) + c.y) + dd.y) / 4.f, (((a.z + bb.z) + c.z) + dd.z) / 4.f,
                    (((a.w + bb.w) + c.w) + dd.w) / 4.f);
}

// one thread per output voxel (b, z, y, x) (x fastest).  p [B, D, H, W, 128]: column 16 dz + o of depth slice d holds that
// slice's 7 x 7 products with the mask weights of kernel depth dz, column 112 + d its products with the occlusion weights
// of input depth d.  logits[o] = (sum over dz of p[z + dz - 3, 16 dz + o], depths outside skipped) + bias[o]; mask =
// softmax; deformation = sum over k of mask[k] * motion_k.  The threads of depth 0 also write the occlusion map.
__global__ void __launch_bounds__(THREADS) combine_kernel(const float* __restrict__ p, const float* __restrict__ mask_bias,
                                                          const float* __restrict__ occ_bias, const float* __restrict__ kd,
                                                          const float* __restrict__ ks, float* __restrict__ mask,
                                                          float* __restrict__ deform, float* __restrict__ occ, int d, int h,
                                                          int w) {
    const int hw = h * w, i = blockIdx.x * THREADS + threadIdx.x, z = blockIdx.y, b = blockIdx.z;
    if (i >= hw) return;
    const int y = i / w, x = i - y * w;
    const float* pb = p + (int64_t)b * d * hw * P_COLS + (int64_t)i * P_COLS;
    float l[NK];
#pragma unroll
    for (int o = 0; o < NK; ++o) l[o] = 0.f;
#pragma unroll
    for (int dz = 0; dz < MASK_TAPS; ++dz) {
        const int zz = z + dz - MASK_TAPS / 2;
        if (zz < 0 || zz >= d) continue;
        const float4* src = reinterpret_cast<const float4*>(pb + (int64_t)zz * hw * P_COLS + dz * NK);
#pragma unroll
        for (int q = 0; q < NK / 4; ++q) {
            const float4 v = __ldg(src + q);
            l[4 * q] += v.x, l[4 * q + 1] += v.y, l[4 * q + 2] += v.z, l[4 * q + 3] += v.w;
        }
    }
    float m = -INFINITY;
#pragma unroll
    for (int o = 0; o < NK; ++o) l[o] += __ldg(mask_bias + o), m = fmaxf(m, l[o]);
    float s = 0.f;
#pragma unroll
    for (int o = 0; o < NK; ++o) l[o] = expf(l[o] - m), s += l[o];
    const float gx = 2.f * ((float)x / (float)(w - 1)) - 1.f, gy = 2.f * ((float)y / (float)(h - 1)) - 1.f,
                gz = 2.f * ((float)z / (float)(d - 1)) - 1.f;
    float fx = 0.f, fy = 0.f, fz = 0.f;
    const float* kdb = kd + b * NKP * 3;
    const float* ksb = ks + b * NKP * 3;
#pragma unroll
    for (int k = 0; k < NK; ++k) {
        const float mk = l[k] / s;
        mask[(((int64_t)b * NK + k) * d + z) * hw + i] = mk;
        float mx = gx, my = gy, mz = gz;
        if (k > 0)
            mx = (gx - __ldg(kdb + 3 * (k - 1))) + __ldg(ksb + 3 * (k - 1)),
            my = (gy - __ldg(kdb + 3 * (k - 1) + 1)) + __ldg(ksb + 3 * (k - 1) + 1),
            mz = (gz - __ldg(kdb + 3 * (k - 1) + 2)) + __ldg(ksb + 3 * (k - 1) + 2);
        fx = fmaf(mk, mx, fx), fy = fmaf(mk, my, fy), fz = fmaf(mk, mz, fz);
    }
    float* df = deform + ((((int64_t)b * d + z) * h + y) * w + x) * 3;
    df[0] = fx, df[1] = fy, df[2] = fz;
    if (z == 0) {
        float a = 0.f;
        for (int zz = 0; zz < d; ++zz) a += __ldg(pb + (int64_t)zz * hw * P_COLS + OCC_COL + zz);
        occ[(int64_t)b * hw + i] = 1.f / (1.f + expf(-(a + __ldg(occ_bias))));
    }
}

// one thread per (output voxel (b, y, x, z), channel quad q), q fastest: vol [B, H, W, D, 32] sampled at deform[b, z, y, x]
// into out [B, H, W, D, 32] (as float4s: element i of out is thread i's)
__global__ void __launch_bounds__(THREADS) warp_kernel(const float4* __restrict__ vol, const float* __restrict__ deform,
                                                       float4* __restrict__ out, int d, int h, int w, int64_t total) {
    const int64_t i = (int64_t)blockIdx.x * THREADS + threadIdx.x;
    if (i >= total) return;
    constexpr int Q = CF / 4;
    const int q = (int)(i % Q);
    int64_t r = i / Q;
    const int z = (int)(r % d);
    r /= d;
    const int x = (int)(r % w);
    r /= w;
    const int y = (int)(r % h);
    const int64_t b = r / h;
    const float* df = deform + (((b * d + z) * h + y) * w + x) * 3;
    const int64_t sx = (int64_t)d * Q;
    out[i] = sample(vol + b * h * w * sx + q, Q, w * sx, sx, __ldg(df), __ldg(df + 1), __ldg(df + 2), d, h, w);
}

}  // namespace v2vdm

extern "C" int e4s_vid2vid_compress_f32(const float* x, const float* wb, float* y, int batch, int d, int h, int w, void* stream) {
    E4S_REQUIRE(x && wb && y, E4S_ERR_ARG);
    E4S_REQUIRE(batch > 0 && batch <= 65535 && d > 0 && h > 0 && w > 0 && (int64_t)d * h * w * v2vdm::CF < (1ll << 31),
                E4S_ERR_SHAPE);
    E4S_REQUIRE(e4s_aligned16(y), E4S_ERR_ALIGN);
    const int nvox = d * h * w;
    v2vdm::compress_kernel<<<dim3((unsigned)e4s_ceil_div(nvox, v2vdm::THREADS), (unsigned)batch), v2vdm::THREADS, 0,
                             (cudaStream_t)stream>>>(x, wb, y, nvox);
    return e4s_launch_status();
}

extern "C" int e4s_vid2vid_motion_input_f32(const float* comp, const float* kp_driving, const float* kp_source, float* y, int y_vp,
                                            int batch, int d, int h, int w, void* stream) {
    E4S_REQUIRE(comp && kp_driving && kp_source && y, E4S_ERR_ARG);
    E4S_REQUIRE(y_vp >= v2vdm::IN_PAD, E4S_ERR_ARG);
    E4S_REQUIRE(batch > 0 && batch <= 65535 && d > 1 && d <= 65535 && h > 1 && w > 1 && (int64_t)d * h * w * y_vp < (1ll << 31),
                E4S_ERR_SHAPE);
    E4S_REQUIRE((y_vp % 4) == 0 && e4s_aligned16(comp) && e4s_aligned16(y), E4S_ERR_ALIGN);
    const dim3 grid((unsigned)e4s_ceil_div((int64_t)h * w, v2vdm::THREADS), (unsigned)d, (unsigned)batch);
    v2vdm::motion_input_kernel<<<grid, v2vdm::THREADS, 0, (cudaStream_t)stream>>>(reinterpret_cast<const float4*>(comp), kp_driving,
                                                                                  kp_source, y, y_vp, d, h, w);
    return e4s_launch_status();
}

extern "C" int e4s_avgpool2_vox_f32(const float* x, float* y, int y_vp, int batch, int h, int w, int d, int c, void* stream) {
    E4S_REQUIRE(x && y && y_vp >= c, E4S_ERR_ARG);
    E4S_REQUIRE(batch > 0 && h > 1 && w > 1 && d > 0 && c > 0 && (h % 2) == 0 && (w % 2) == 0 && (c % 4) == 0, E4S_ERR_SHAPE);
    E4S_REQUIRE((y_vp % 4) == 0 && e4s_aligned16(x) && e4s_aligned16(y), E4S_ERR_ALIGN);
    const int64_t total4 = (int64_t)batch * (h / 2) * (w / 2) * d * (c / 4);
    v2vdm::avgpool2_vox_kernel<<<(unsigned)e4s_ceil_div(total4, v2vdm::THREADS), v2vdm::THREADS, 0, (cudaStream_t)stream>>>(
        x, y, total4, h, w, d, c / 4, y_vp);
    return e4s_launch_status();
}

extern "C" int e4s_vid2vid_warp_f32(const float* vol, const float* deformation, float* y, int batch, int d, int h, int w,
                                     void* stream) {
    E4S_REQUIRE(vol && deformation && y, E4S_ERR_ARG);
    E4S_REQUIRE(batch > 0 && d > 0 && h > 0 && w > 0 && (int64_t)d * h * w * v2vdm::CF < (1ll << 31), E4S_ERR_SHAPE);
    E4S_REQUIRE(e4s_aligned16(vol) && e4s_aligned16(y), E4S_ERR_ALIGN);
    const int64_t total = (int64_t)batch * d * h * w * (v2vdm::CF / 4);
    v2vdm::warp_kernel<<<(unsigned)e4s_ceil_div(total, v2vdm::THREADS), v2vdm::THREADS, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<const float4*>(vol), deformation, reinterpret_cast<float4*>(y), d, h, w, total);
    return e4s_launch_status();
}

extern "C" int e4s_vid2vid_motion_combine_f32(const float* p, const float* mask_bias, const float* occ_bias,
                                              const float* kp_driving, const float* kp_source, float* mask, float* deformation,
                                              float* occlusion, int batch, int d, int h, int w, void* stream) {
    E4S_REQUIRE(p && mask_bias && occ_bias && kp_driving && kp_source && mask && deformation && occlusion, E4S_ERR_ARG);
    E4S_REQUIRE(batch > 0 && batch <= 65535 && d > 1 && d <= v2vdm::P_COLS - v2vdm::OCC_COL && h > 1 && w > 1, E4S_ERR_SHAPE);
    E4S_REQUIRE(e4s_aligned16(p), E4S_ERR_ALIGN);
    const dim3 grid((unsigned)e4s_ceil_div((int64_t)h * w, v2vdm::THREADS), (unsigned)d, (unsigned)batch);
    v2vdm::combine_kernel<<<grid, v2vdm::THREADS, 0, (cudaStream_t)stream>>>(p, mask_bias, occ_bias, kp_driving, kp_source, mask,
                                                                             deformation, occlusion, d, h, w);
    return e4s_launch_status();
}
