// Mask / index operations (bit-exact) and layout shuffles.
//
// The reference carries region masks as float one-hot tensors [B, ncls, H, W] and multiplies conv
// outputs by them (src/models/stylegan2/model.py:391-398, 430-437).  Here a mask becomes a uint8
// label map [B, H, W] plus a nearest-resized label pyramid: 1 byte per pixel instead of 4*ncls,
// and the per-region sum turns into a per-pixel selection (bit-identical for one-hot masks,
// SURVEY.md App. A).
#include "common.cuh"

namespace {

__global__ void __launch_bounds__(256) onehot_to_label_kernel(const float* __restrict__ onehot,
                                                              uint8_t* __restrict__ label, int* __restrict__ flag,
                                                              int ncls, int64_t hw, int64_t total) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        int64_t b = i / hw, p = i - b * hw;
        const float* src = onehot + b * ncls * hw + p;
        int best = 0, ones = 0;
        bool clean = true;
        for (int c = 0; c < ncls; ++c) {
            float v = src[(int64_t)c * hw];
            if (v == 1.0f) {
                if (ones == 0) best = c;
                ++ones;
            } else if (v != 0.0f) {
                clean = false;
            }
        }
        if (!clean || ones != 1) *flag = 1;  // benign race: every writer stores 1
        label[i] = (uint8_t)best;
    }
}

__global__ void __launch_bounds__(256) label_to_onehot_kernel(const uint8_t* __restrict__ label,
                                                              float* __restrict__ onehot, int ncls, int64_t hw,
                                                              int64_t total) {
    // total = B * ncls * hw output elements; consecutive threads -> consecutive pixels of one class plane
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        int64_t p = i % hw;
        int64_t t = i / hw;
        int c = (int)(t % ncls);
        int64_t b = t / ncls;
        onehot[i] = (label[b * hw + p] == c) ? 1.0f : 0.0f;
    }
}

__global__ void __launch_bounds__(256) label_resize_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst,
                                                           int in_h, int in_w, int out_h, int out_w, float sy, float sx,
                                                           int64_t total) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        int ox = (int)(i % out_w);
        int64_t t = i / out_w;
        int oy = (int)(t % out_h);
        int64_t b = t / out_h;
        // ATen nearest_neighbor_compute_source_index: min(floorf(dst * scale), in - 1)
        int iy = min((int)floorf(oy * sy), in_h - 1);
        int ix = min((int)floorf(ox * sx), in_w - 1);
        dst[i] = src[(b * in_h + iy) * in_w + ix];
    }
}

__global__ void __launch_bounds__(256) label_remap_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst,
                                                          const uint8_t* __restrict__ lut, int64_t n) {
    __shared__ uint8_t s_lut[256];
    s_lut[threadIdx.x] = lut[threadIdx.x];
    __syncthreads();
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        dst[i] = s_lut[src[i]];
}

// ---- face-swapping mask stage (SURVEY.md section 8f.3), bit-exact --------------------------------------------------
// Shape swapping of two 12-class parsing maps: swap_head_mask_revisit_considerGlass, src/utils/swap_face_mask.py:33-83.
// The reference applies ~15 masked assignments over whole arrays on the CPU; every pixel is independent and later
// assignments override earlier ones, so the sequence is one decision list per pixel.
__device__ __forceinline__ void swap_head_pixel(int s, int t, int hair_first, uint8_t& res, uint8_t& hole, uint8_t& fg) {
    int r = 0;
    if (t == 0) r = 99;                                       // :42 place-holder for the target's background
    else if (t == 8 || t == 7 || t == 11) r = t;              // :43-45 neck, ear, ear rings of the target
    if (hair_first && t == 4) r = 4;                          // :47-48
    if (r != 99 && (s == 1 || s == 2 || s == 3 || s == 5 || s == 6 || s == 9)) r = s;   // :51-56 inner face of the source
    if (!hair_first && t == 4) r = 4;                         // :66-67
    if (t == 10) r = 10;                                      // :70 eye glasses of the target
    const bool is_hole = r == 0;                              // :74-78
    if (is_hole) r = 6;                                       // missing pixels become skin
    if (r == 99) r = 0;                                       // :81
    res = (uint8_t)r;
    hole = is_hole ? 255 : 0;
    // scripts/face_swap.py:280-284: background = {0, 11, 4}; holes count as foreground
    fg = (uint8_t)((!(r == 0 || r == 11 || r == 4)) || is_hole);
}

__global__ void __launch_bounds__(256) swap_head_mask_kernel(const uint8_t* __restrict__ src, const uint8_t* __restrict__ tgt,
                                                             uint8_t* __restrict__ res, uint8_t* __restrict__ hole,
                                                             uint8_t* __restrict__ fg, int64_t n, int hair_first, int vec) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    if (vec) {                                                // 16 labels per thread and step, 128-bit accesses
        const int64_t n16 = n >> 4;
        for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n16; i += stride) {
            const uint4 sv = __ldg(reinterpret_cast<const uint4*>(src) + i), tv = __ldg(reinterpret_cast<const uint4*>(tgt) + i);
            const uint32_t sw[4] = {sv.x, sv.y, sv.z, sv.w}, tw[4] = {tv.x, tv.y, tv.z, tv.w};
            uint32_t rw[4], hw[4], fw[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                rw[k] = hw[k] = fw[k] = 0;
#pragma unroll
                for (int b = 0; b < 4; ++b) {
                    uint8_t r, h, f;
                    swap_head_pixel((sw[k] >> (8 * b)) & 255, (tw[k] >> (8 * b)) & 255, hair_first, r, h, f);
                    rw[k] |= (uint32_t)r << (8 * b), hw[k] |= (uint32_t)h << (8 * b), fw[k] |= (uint32_t)f << (8 * b);
                }
            }
            reinterpret_cast<uint4*>(res)[i] = make_uint4(rw[0], rw[1], rw[2], rw[3]);
            reinterpret_cast<uint4*>(hole)[i] = make_uint4(hw[0], hw[1], hw[2], hw[3]);
            if (fg) reinterpret_cast<uint4*>(fg)[i] = make_uint4(fw[0], fw[1], fw[2], fw[3]);
        }
    }
    const int64_t done = vec ? (n >> 4) << 4 : 0;
    for (int64_t i = done + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        uint8_t r, h, f;
        swap_head_pixel(src[i], tgt[i], hair_first, r, h, f);
        res[i] = r, hole[i] = h;
        if (fg) fg[i] = f;
    }
}

// Flat (2r+1)^2 box dilation (MAXOP) / erosion of uint8 masks with the 'geodesic' border of the reference
// (src/utils/morphology.py:83-86, 170-173: positions outside the image never win).  The reference turns the window
// into (2r+1)^2 = 121 convolution channels and reduces over them; a box is separable, so one CTA stages a 32x64 tile
// with its halo, reduces along rows in shared memory, then along columns.
constexpr int MT_W = 64, MT_H = 32, MORPH_MAX_R = 16;
template <typename T, bool MAXOP>
__global__ void __launch_bounds__(256) box_morph_kernel(const T* __restrict__ src, T* __restrict__ dst, int h, int w,
                                                        int radius, T neutral) {
    __shared__ T raw[(MT_H + 2 * MORPH_MAX_R) * (MT_W + 2 * MORPH_MAX_R)];
    __shared__ T rows[(MT_H + 2 * MORPH_MAX_R) * MT_W];
    const int x0 = blockIdx.x * MT_W, y0 = blockIdx.y * MT_H;
    const T* sp = src + (int64_t)blockIdx.z * h * w;
    const int sw = MT_W + 2 * radius, sh = MT_H + 2 * radius;
    for (int i = threadIdx.x; i < sw * sh; i += 256) {
        const int ry = i / sw, rx = i - ry * sw;
        const int gy = y0 - radius + ry, gx = x0 - radius + rx;
        raw[i] = (gy >= 0 && gy < h && gx >= 0 && gx < w) ? sp[(int64_t)gy * w + gx] : neutral;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < sh * MT_W; i += 256) {
        const int ry = i / MT_W, cx = i - ry * MT_W;
        const T* rp = raw + ry * sw + cx;
        T v = rp[0];
        for (int k = 1; k <= 2 * radius; ++k) v = MAXOP ? max(v, rp[k]) : min(v, rp[k]);
        rows[i] = v;
    }
    __syncthreads();
    T* dp = dst + (int64_t)blockIdx.z * h * w;
    for (int i = threadIdx.x; i < MT_H * MT_W; i += 256) {
        const int cy = i / MT_W, cx = i - cy * MT_W;
        const int gy = y0 + cy, gx = x0 + cx;
        if (gy >= h || gx >= w) continue;
        T v = rows[cy * MT_W + cx];
        for (int k = 1; k <= 2 * radius; ++k) v = MAXOP ? max(v, rows[(cy + k) * MT_W + cx]) : min(v, rows[(cy + k) * MT_W + cx]);
        dp[(int64_t)gy * w + gx] = v;
    }
}

template <typename T>
int launch_box_morph(const T* src, T* dst, int planes, int h, int w, int radius, int erode, T lo, T hi, cudaStream_t st) {
    E4S_REQUIRE(src && dst && src != dst && planes > 0 && h > 0 && w > 0 && radius >= 0, E4S_ERR_ARG);
    E4S_REQUIRE(radius <= MORPH_MAX_R && planes <= 65535, E4S_ERR_SHAPE);
    dim3 grid((unsigned)e4s_ceil_div(w, MT_W), (unsigned)e4s_ceil_div(h, MT_H), (unsigned)planes);
    E4S_REQUIRE(grid.y <= 65535, E4S_ERR_SHAPE);
    if (erode)
        box_morph_kernel<T, false><<<grid, 256, 0, st>>>(src, dst, h, w, radius, hi);
    else
        box_morph_kernel<T, true><<<grid, 256, 0, st>>>(src, dst, h, w, radius, lo);
    return e4s_launch_status();
}

// Region mean: grid (channel chunks of 32, B).  Each warp walks pixels; lane = channel inside the
// 32-channel chunk (pixel-major: the 32 lanes read 128 contiguous bytes).  Per-class partial sums
// live in shared memory [ncls][32] per warp, reduced across warps at the end.  Area counts are
// integers; sum order is fixed -> deterministic.
constexpr int RM_WARPS = 8;
__global__ void __launch_bounds__(32 * RM_WARPS) region_mean_kernel(const float* __restrict__ feats,
                                                                     const uint8_t* __restrict__ label,
                                                                     float* __restrict__ out, int* __restrict__ area,
                                                                     int ncls, int hw, int c) {
    extern __shared__ float sm[];  // [RM_WARPS][ncls][32] sums, then [RM_WARPS][ncls] counts (as int)
    float* sums = sm;
    int* cnts = reinterpret_cast<int*>(sm + RM_WARPS * ncls * 32);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int b = blockIdx.y, ch = blockIdx.x * 32 + lane;
    for (int i = threadIdx.x; i < RM_WARPS * ncls * 32; i += blockDim.x) sums[i] = 0.f;
    for (int i = threadIdx.x; i < RM_WARPS * ncls; i += blockDim.x) cnts[i] = 0;
    __syncthreads();
    const float* fb = feats + (int64_t)b * hw * c;
    const uint8_t* lb = label + (int64_t)b * hw;
    float* my = sums + warp * ncls * 32;
    int* myc = cnts + warp * ncls;
    for (int p = warp; p < hw; p += RM_WARPS) {
        int cls = lb[p];
        if (cls >= ncls) continue;
        if (ch < c) my[cls * 32 + lane] += fb[(int64_t)p * c + ch];
        if (lane == 0) myc[cls] += 1;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < ncls * 32; i += blockDim.x) {
        int cls = i >> 5, l = i & 31;
        float s = 0.f;
        int n = 0;
        for (int w = 0; w < RM_WARPS; ++w) s += sums[w * ncls * 32 + i], n += cnts[w * ncls + cls];
        int chn = blockIdx.x * 32 + l;
        if (chn < c) out[((int64_t)b * ncls + cls) * c + chn] = n > 0 ? s / (float)n : 0.f;
        if (blockIdx.x == 0 && l == 0) area[b * ncls + cls] = n;
    }
}

// Tiled transpose between planar [B, C, HW] and pixel-major [B, HW, C].
__global__ void __launch_bounds__(256) transpose_kernel(const float* __restrict__ src, float* __restrict__ dst,
                                                        int rows, int cols) {
    // src: [batch][rows][cols] -> dst: [batch][cols][rows]
    __shared__ float t[32][33];
    const int b = blockIdx.z;
    const float* s = src + (int64_t)b * rows * cols;
    float* d = dst + (int64_t)b * rows * cols;
    int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
    int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    for (int j = ty; j < 32; j += 8) {
        int r = r0 + j, c = c0 + tx;
        if (r < rows && c < cols) t[j][tx] = s[(int64_t)r * cols + c];
    }
    __syncthreads();
    for (int j = ty; j < 32; j += 8) {
        int c = c0 + j, r = r0 + tx;
        if (r < rows && c < cols) d[(int64_t)c * rows + r] = t[tx][j];
    }
}

inline unsigned gs_grid(int64_t total) {
    int64_t want = e4s_ceil_div(total, 256), cap = (int64_t)E4S_NUM_SMS * 16;
    if (want < 1) want = 1;
    return (unsigned)(want < cap ? want : cap);
}

}  // namespace

extern "C" int e4s_onehot_to_label_u8(const float* onehot, uint8_t* label, int* flag, int batch, int ncls, int h, int w,
                                      void* stream) {
    E4S_REQUIRE(onehot && label && flag && batch > 0 && ncls > 0 && ncls <= 255 && h > 0 && w > 0, E4S_ERR_ARG);
    int64_t hw = (int64_t)h * w, total = hw * batch;
    onehot_to_label_kernel<<<gs_grid(total), 256, 0, (cudaStream_t)stream>>>(onehot, label, flag, ncls, hw, total);
    return e4s_launch_status();
}

extern "C" int e4s_label_to_onehot_f32(const uint8_t* label, float* onehot, int batch, int ncls, int h, int w,
                                       void* stream) {
    E4S_REQUIRE(onehot && label && batch > 0 && ncls > 0 && ncls <= 255 && h > 0 && w > 0, E4S_ERR_ARG);
    int64_t hw = (int64_t)h * w, total = hw * batch * ncls;
    label_to_onehot_kernel<<<gs_grid(total), 256, 0, (cudaStream_t)stream>>>(label, onehot, ncls, hw, total);
    return e4s_launch_status();
}

extern "C" int e4s_label_resize_nearest_u8(const uint8_t* src, uint8_t* dst, int batch, int in_h, int in_w, int out_h,
                                           int out_w, void* stream) {
    E4S_REQUIRE(src && dst && batch > 0 && in_h > 0 && in_w > 0 && out_h > 0 && out_w > 0, E4S_ERR_ARG);
    float sy = (float)in_h / (float)out_h, sx = (float)in_w / (float)out_w;
    int64_t total = (int64_t)batch * out_h * out_w;
    label_resize_kernel<<<gs_grid(total), 256, 0, (cudaStream_t)stream>>>(src, dst, in_h, in_w, out_h, out_w, sy, sx,
                                                                           total);
    return e4s_launch_status();
}

extern "C" int e4s_label_remap_u8(const uint8_t* src, uint8_t* dst, const uint8_t* lut256, int64_t n, void* stream) {
    E4S_REQUIRE(src && dst && lut256 && n > 0, E4S_ERR_ARG);
    label_remap_kernel<<<gs_grid(n), 256, 0, (cudaStream_t)stream>>>(src, dst, lut256, n);
    return e4s_launch_status();
}

extern "C" int e4s_swap_head_mask_u8(const uint8_t* source, const uint8_t* target, uint8_t* swapped, uint8_t* hole,
                                     uint8_t* foreground, int64_t n, int hair_first, void* stream) {
    E4S_REQUIRE(source && target && swapped && hole && n > 0, E4S_ERR_ARG);
    const int vec = e4s_aligned16(source) && e4s_aligned16(target) && e4s_aligned16(swapped) && e4s_aligned16(hole) &&
                    (!foreground || e4s_aligned16(foreground));
    swap_head_mask_kernel<<<gs_grid(vec ? e4s_ceil_div(n, 16) : n), 256, 0, (cudaStream_t)stream>>>(
        source, target, swapped, hole, foreground, n, hair_first ? 1 : 0, vec);
    return e4s_launch_status();
}

extern "C" int e4s_mask_box_morph_u8(const uint8_t* src, uint8_t* dst, int planes, int h, int w, int radius, int erode,
                                     void* stream) {
    return launch_box_morph<uint8_t>(src, dst, planes, h, w, radius, erode, 0, 255, (cudaStream_t)stream);
}

extern "C" int e4s_box_morph_f32(const float* src, float* dst, int planes, int h, int w, int radius, int erode, float max_val,
                                 void* stream) {
    // the reference pads with -max_val (dilation) / +max_val (erosion): morphology.py:83-86, 170-173
    return launch_box_morph<float>(src, dst, planes, h, w, radius, erode, -max_val, max_val, (cudaStream_t)stream);
}

extern "C" int e4s_region_mean_f32(const float* feats, const uint8_t* label, float* out, int* area, int batch, int ncls,
                                   int h, int w, int c, void* stream) {
    E4S_REQUIRE(feats && label && out && area && batch > 0 && ncls > 0 && h > 0 && w > 0 && c > 0, E4S_ERR_ARG);
    E4S_REQUIRE(ncls <= 64, E4S_ERR_SHAPE);
    dim3 grid((unsigned)e4s_ceil_div(c, 32), batch);
    size_t smem = (size_t)RM_WARPS * ncls * 32 * sizeof(float) + (size_t)RM_WARPS * ncls * sizeof(int);   // > 48 KB from ncls 47
    static E4sSmemOptIn optin;
    if (const int rc = e4s_smem_optin(optin, region_mean_kernel, smem)) return rc;
    region_mean_kernel<<<grid, 32 * RM_WARPS, smem, (cudaStream_t)stream>>>(feats, label, out, area, ncls, h * w, c);
    return e4s_launch_status();
}

extern "C" int e4s_planar_to_pixel_f32(const float* x, float* y, int batch, int c, int h, int w, void* stream) {
    E4S_REQUIRE(x && y && batch > 0 && c > 0 && h > 0 && w > 0, E4S_ERR_ARG);
    int hw = h * w;
    dim3 grid((unsigned)e4s_ceil_div(hw, 32), (unsigned)e4s_ceil_div(c, 32), batch);
    transpose_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(x, y, c, hw);
    return e4s_launch_status();
}

extern "C" int e4s_pixel_to_planar_f32(const float* x, float* y, int batch, int c, int h, int w, void* stream) {
    E4S_REQUIRE(x && y && batch > 0 && c > 0 && h > 0 && w > 0, E4S_ERR_ARG);
    int hw = h * w;
    dim3 grid((unsigned)e4s_ceil_div(c, 32), (unsigned)e4s_ceil_div(hw, 32), batch);
    transpose_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(x, y, hw, c);
    return e4s_launch_status();
}
