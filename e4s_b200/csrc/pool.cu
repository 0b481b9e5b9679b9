// Average-pooling pyramid for the inversion loop's loss networks (sm_90a, HBM-bound streaming kernels).
//
// scripts/optimization.py:103-110 evaluates LPIPS on adaptive_avg_pool2d(img, 1024 / 2^i), i = 0..2; the identity loss pools
// to 256x256 (src/criteria/id_loss.py:14,26) and the parsing loss to 512x512 (src/criteria/face_parsing/face_parsing_loss.py:25,47).
// For a 1024x1024 image every one of those is a 2x2 or 4x4 block mean, so ONE pass over the image produces the half- and
// quarter-resolution copies all three loss networks start from (the reference launches five pooling kernels per image and
// reads the 1024x1024 tensor five times), and ONE pass brings their three gradients back to full resolution.
#include "common.cuh"

namespace {

// one thread = one 4x4 input block: four 128-bit loads, two 64-bit stores (half resolution), one scalar store (quarter)
__global__ void __launch_bounds__(256) avgpool_pyramid_kernel(const float* __restrict__ x, float* __restrict__ y2, float* __restrict__ y4,
                                                              int64_t planes, int h, int w) {
    const int w4 = w >> 2, h4 = h >> 2;
    const int64_t total = planes * h4 * w4;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int bx = (int)(i % w4);
        const int by = (int)((i / w4) % h4);
        const int64_t pl = i / ((int64_t)w4 * h4);
        const float* src = x + (pl * h + 4 * by) * (int64_t)w + 4 * bx;
        const float4 r0 = ld_stream_f4(src), r1 = ld_stream_f4(src + w), r2 = ld_stream_f4(src + 2 * (int64_t)w), r3 = ld_stream_f4(src + 3 * (int64_t)w);
        const float a = 0.25f * ((r0.x + r0.y) + (r1.x + r1.y)), b = 0.25f * ((r0.z + r0.w) + (r1.z + r1.w));
        const float c = 0.25f * ((r2.x + r2.y) + (r3.x + r3.y)), d = 0.25f * ((r2.z + r2.w) + (r3.z + r3.w));
        float* d2 = y2 + (pl * (h >> 1) + 2 * by) * (int64_t)(w >> 1) + 2 * bx;
        *reinterpret_cast<float2*>(d2) = make_float2(a, b);
        *reinterpret_cast<float2*>(d2 + (w >> 1)) = make_float2(c, d);
        y4[(pl * h4 + by) * (int64_t)w4 + bx] = 0.25f * ((a + b) + (c + d));
    }
}

// gx = g1 + up2(g2) / 4 + up4(g4) / 16 (any of the three may be absent)
__global__ void __launch_bounds__(256) avgpool_pyramid_bwd_kernel(const float* __restrict__ g1, const float* __restrict__ g2,
                                                                  const float* __restrict__ g4, float* __restrict__ gx, int64_t planes,
                                                                  int h, int w) {
    const int w4 = w >> 2, h4 = h >> 2;
    const int64_t total = planes * h4 * w4;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int bx = (int)(i % w4);
        const int by = (int)((i / w4) % h4);
        const int64_t pl = i / ((int64_t)w4 * h4);
        const float q = g4 ? 0.0625f * g4[(pl * h4 + by) * (int64_t)w4 + bx] : 0.f;
        float2 t = make_float2(0.f, 0.f), u = make_float2(0.f, 0.f);
        if (g2) {
            const float* s2 = g2 + (pl * (h >> 1) + 2 * by) * (int64_t)(w >> 1) + 2 * bx;
            t = *reinterpret_cast<const float2*>(s2);
            u = *reinterpret_cast<const float2*>(s2 + (w >> 1));
        }
        const float a = 0.25f * t.x + q, b = 0.25f * t.y + q, c = 0.25f * u.x + q, d = 0.25f * u.y + q;
        const int64_t off = (pl * h + 4 * by) * (int64_t)w + 4 * bx;
        float4 o[4] = {make_float4(a, a, b, b), make_float4(a, a, b, b), make_float4(c, c, d, d), make_float4(c, c, d, d)};
        if (g1) {
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                const float4 v = ld_stream_f4(g1 + off + r * (int64_t)w);
                o[r].x += v.x, o[r].y += v.y, o[r].z += v.z, o[r].w += v.w;
            }
        }
#pragma unroll
        for (int r = 0; r < 4; ++r) st_stream_f4(gx + off + r * (int64_t)w, o[r]);
    }
}

int grid_for(int64_t total) {
    int64_t want = e4s_ceil_div(total, 256);
    const int64_t cap = (int64_t)e4s_num_sms() * 16;
    return (int)(want < cap ? (want < 1 ? 1 : want) : cap);
}

}  // namespace

extern "C" int e4s_avgpool_pyramid_f32(const float* x, float* y2, float* y4, long long planes, int h, int w, void* stream) {
    E4S_REQUIRE(x && y2 && y4 && planes > 0 && h > 0 && w > 0, E4S_ERR_ARG);
    E4S_REQUIRE((h % 4) == 0 && (w % 8) == 0, E4S_ERR_SHAPE);                    // 128-bit loads, 64-bit stores
    E4S_REQUIRE(e4s_aligned16(x) && (reinterpret_cast<uintptr_t>(y2) & 7) == 0, E4S_ERR_ALIGN);
    const int64_t total = (int64_t)planes * (h / 4) * (w / 4);
    avgpool_pyramid_kernel<<<grid_for(total), 256, 0, (cudaStream_t)stream>>>(x, y2, y4, planes, h, w);
    return e4s_launch_status();
}

extern "C" int e4s_avgpool_pyramid_bwd_f32(const float* g1, const float* g2, const float* g4, float* gx, long long planes, int h,
                                           int w, void* stream) {
    E4S_REQUIRE(gx && (g1 || g2 || g4) && planes > 0 && h > 0 && w > 0, E4S_ERR_ARG);
    E4S_REQUIRE((h % 4) == 0 && (w % 8) == 0, E4S_ERR_SHAPE);
    E4S_REQUIRE(e4s_aligned16(gx) && (!g1 || e4s_aligned16(g1)) && (!g2 || (reinterpret_cast<uintptr_t>(g2) & 7) == 0), E4S_ERR_ALIGN);
    const int64_t total = (int64_t)planes * (h / 4) * (w / 4);
    avgpool_pyramid_bwd_kernel<<<grid_for(total), 256, 0, (cudaStream_t)stream>>>(g1, g2, g4, gx, planes, h, w);
    return e4s_launch_status();
}
