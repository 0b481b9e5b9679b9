// The data-dependent tail of GPEN's RetinaFace-R50 detector (src/pretrained/gpen/face_detect/retinaface_detection.py:61-131)
// and its input conversion, around the tensor-core convolutions that run the network:
//   * prep: planar BGR uint8 / fp32 pixels minus the detector's mean (104, 117, 123);
//   * decode: per prior, the two-way softmax, PriorBox's anchor (computed here, in double as prior_box.py does, then
//     rounded to float: no prior table), decode / decode_landm (box_utils.py:209-247) and the scale to pixels, in the
//     reference's fp32 operation order with no FMA contraction;
//   * NMS: one CTA per image walks the candidates in sorted order with py_cpu_nms's fp32 arithmetic (greedy; a candidate
//     survives only if its overlap with every kept box is <= the threshold, so a NaN overlap suppresses, as in numpy) and
//     writes up to keep_top_k detections and their count.  No host synchronisation: the whole tail can be graph-captured.
#include "common.cuh"

namespace retina {

constexpr int NLEVEL = 3, NANCHOR = 2, HEAD_CH = 32;      // head channels: class 4 | bbox 8 | landmark 20
__device__ __constant__ int STEPS[NLEVEL] = {8, 16, 32};
__device__ __constant__ int MIN_SIZES[NLEVEL][NANCHOR] = {{16, 32}, {64, 128}, {256, 512}};

__global__ void prep_kernel(const void* __restrict__ x, int x_u8, float* __restrict__ y, int64_t hw, int64_t total) {
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= total) return;
    const int c = (int)((i / hw) % 3);
    const float v = x_u8 ? (float)static_cast<const uint8_t*>(x)[i] : static_cast<const float*>(x)[i];
    y[i] = __fsub_rn(v, c == 0 ? 104.f : c == 1 ? 117.f : 123.f);
}

// One thread per prior (b, level, row, column, anchor), in the reference's prior order.
__global__ void decode_kernel(const float* __restrict__ heads, int batch, int h, int w, float resize, float conf_thr,
                              float* __restrict__ boxes, float* __restrict__ landms, float* __restrict__ keys,
                              float* __restrict__ loc, float* __restrict__ conf, float* __restrict__ landm_raw,
                              int num_priors) {
    const int64_t gid = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (gid >= (int64_t)batch * num_priors) return;
    const int b = (int)(gid / num_priors);
    int pr = (int)(gid % num_priors);
    // level, pixel and anchor of the prior; level l's head map sits after the maps of the levels before it
    int64_t base = 0;
    int lvl = 0, lh = h / STEPS[0], lw = w / STEPS[0];
    while (pr >= lh * lw * NANCHOR) {
        pr -= lh * lw * NANCHOR;
        base += (int64_t)batch * lh * lw * HEAD_CH;
        ++lvl;
        lh = h / STEPS[lvl], lw = w / STEPS[lvl];
    }
    const int a = pr % NANCHOR, pix = pr / NANCHOR, i = pix / lw, j = pix % lw;
    const float* hd = heads + base + ((int64_t)b * lh * lw + pix) * HEAD_CH;
    // PriorBox.forward: [cx, cy, s_kx, s_ky] in Python floats, then torch.Tensor (float32)
    const double step = STEPS[lvl], ms = MIN_SIZES[lvl][a];
    const float cx = (float)((j + 0.5) * step / w), cy = (float)((i + 0.5) * step / h);
    const float sw = (float)(ms / w), sh = (float)(ms / h);

    const float c0 = hd[2 * a], c1 = hd[2 * a + 1];
    const float* l = hd + 4 + 4 * a;
    const float* lm = hd + 12 + 10 * a;
    const int64_t o = (int64_t)b * num_priors + (gid % num_priors);
    if (loc)
        for (int k = 0; k < 4; ++k) loc[o * 4 + k] = l[k];
    if (landm_raw)
        for (int k = 0; k < 10; ++k) landm_raw[o * 10 + k] = lm[k];
    // F.softmax over the two logits (as torch's CUDA kernel: exp(x - max) / sum)
    const float mx = fmaxf(c0, c1);
    const float e0 = expf(__fsub_rn(c0, mx)), e1 = expf(__fsub_rn(c1, mx)), s = __fadd_rn(e0, e1);
    const float p0 = __fdiv_rn(e0, s), p1 = __fdiv_rn(e1, s);
    if (conf) conf[o * 2] = p0, conf[o * 2 + 1] = p1;
    if (keys) keys[o] = p1 > conf_thr ? p1 : -INFINITY;
    // decode: centre + loc * 0.1 * size, size * exp(loc * 0.2); corners; then * [W, H, W, H] / resize
    const float fw = (float)w, fh = (float)h;
    if (boxes) {
        const float bx = __fadd_rn(cx, __fmul_rn(__fmul_rn(l[0], 0.1f), sw));
        const float by = __fadd_rn(cy, __fmul_rn(__fmul_rn(l[1], 0.1f), sh));
        const float bw = __fmul_rn(sw, expf(__fmul_rn(l[2], 0.2f)));
        const float bh = __fmul_rn(sh, expf(__fmul_rn(l[3], 0.2f)));
        const float x1 = __fsub_rn(bx, __fdiv_rn(bw, 2.f)), y1 = __fsub_rn(by, __fdiv_rn(bh, 2.f));
        const float x2 = __fadd_rn(bw, x1), y2 = __fadd_rn(bh, y1);
        boxes[o * 4 + 0] = __fdiv_rn(__fmul_rn(x1, fw), resize);
        boxes[o * 4 + 1] = __fdiv_rn(__fmul_rn(y1, fh), resize);
        boxes[o * 4 + 2] = __fdiv_rn(__fmul_rn(x2, fw), resize);
        boxes[o * 4 + 3] = __fdiv_rn(__fmul_rn(y2, fh), resize);
    }
    if (landms)
        for (int k = 0; k < 5; ++k) {
            const float lx = __fadd_rn(cx, __fmul_rn(__fmul_rn(lm[2 * k], 0.1f), sw));
            const float ly = __fadd_rn(cy, __fmul_rn(__fmul_rn(lm[2 * k + 1], 0.1f), sh));
            landms[o * 10 + 2 * k] = __fdiv_rn(__fmul_rn(lx, fw), resize);
            landms[o * 10 + 2 * k + 1] = __fdiv_rn(__fmul_rn(ly, fh), resize);
        }
}

// numpy's maximum / minimum: NaN propagates
__device__ __forceinline__ float np_max(float a, float b) { return a != a ? a : (b != b ? b : fmaxf(a, b)); }
__device__ __forceinline__ float np_min(float a, float b) { return a != a ? a : (b != b ? b : fminf(a, b)); }
// (x2 - x1 + 1) * (y2 - y1 + 1)
__device__ __forceinline__ float area(float4 v) {
    return __fmul_rn(__fadd_rn(__fsub_rn(v.z, v.x), 1.f), __fadd_rn(__fsub_rn(v.w, v.y), 1.f));
}

constexpr int NMS_THREADS = 512;

__global__ void __launch_bounds__(NMS_THREADS) nms_kernel(const float4* __restrict__ boxes, const float* __restrict__ landms,
                                                          const float* __restrict__ keys, const int64_t* __restrict__ order,
                                                          int num_priors, float conf_thr, float nms_thr, int top_k,
                                                          int keep_top_k, float* __restrict__ dets, float* __restrict__ ldm_out,
                                                          int* __restrict__ count) {
    extern __shared__ uint8_t sup[];                  // [min(top_k, P)]: suppressed flags in sorted order
    __shared__ int s_cnt[NMS_THREADS / 32];
    const int b = blockIdx.x, t = threadIdx.x;
    const float* key = keys + (int64_t)b * num_priors;
    const int64_t* od = order + (int64_t)b * num_priors;
    const float4* bx = boxes + (int64_t)b * num_priors;
    const int lim = min(top_k, num_priors);
    // candidates (score > conf_thr) form the sorted prefix; cut to top_k
    int cnt = 0;
    for (int i = t; i < lim; i += NMS_THREADS) {
        cnt += key[i] > conf_thr;
        sup[i] = 0;
    }
    cnt = __reduce_add_sync(0xffffffffu, cnt);
    if ((t & 31) == 0) s_cnt[t >> 5] = cnt;
    __syncthreads();
    int n = 0;
    for (int k = 0; k < NMS_THREADS / 32; ++k) n += s_cnt[k];
    // greedy: every thread walks to the same next unsuppressed candidate (flags are written only past it)
    int i = 0, kept = 0;
    while (kept < keep_top_k) {
        while (i < n && sup[i]) ++i;
        if (i >= n) break;
        const int64_t pi = od[i];
        const float4 bi = bx[pi];
        if (t < 5) dets[((int64_t)b * keep_top_k + kept) * 5 + t] = t < 4 ? (&bi.x)[t] : key[i];
        else if (t < 15) {                            // x1..x5, y1..y5 (detect()'s landmark order)
            const int k = t - 5;
            ldm_out[((int64_t)b * keep_top_k + kept) * 10 + k] = landms[((int64_t)b * num_priors + pi) * 10 + (k % 5) * 2 + k / 5];
        }
        const float ai = area(bi);
        for (int j = i + 1 + t; j < n; j += NMS_THREADS) {
            if (sup[j]) continue;
            const float4 bj = bx[od[j]];
            const float xx1 = np_max(bi.x, bj.x), yy1 = np_max(bi.y, bj.y);
            const float xx2 = np_min(bi.z, bj.z), yy2 = np_min(bi.w, bj.w);
            const float ww = np_max(0.f, __fadd_rn(__fsub_rn(xx2, xx1), 1.f));
            const float hh = np_max(0.f, __fadd_rn(__fsub_rn(yy2, yy1), 1.f));
            const float inter = __fmul_rn(ww, hh);
            const float ovr = __fdiv_rn(inter, __fsub_rn(__fadd_rn(ai, area(bj)), inter));
            if (!(ovr <= nms_thr)) sup[j] = 1;
        }
        __syncthreads();
        ++kept, ++i;
    }
    if (t == 0) count[b] = kept;
}

}  // namespace retina

extern "C" int e4s_retinaface_prep_f32(const void* x, int x_u8, float* y, int batch, int h, int w, void* stream) {
    E4S_REQUIRE(x && y && batch > 0 && h > 0 && w > 0, E4S_ERR_ARG);
    const int64_t total = (int64_t)batch * 3 * h * w;
    retina::prep_kernel<<<(unsigned)e4s_ceil_div(total, 256), 256, 0, (cudaStream_t)stream>>>(x, x_u8, y, (int64_t)h * w, total);
    return e4s_launch_status();
}

extern "C" int e4s_retinaface_decode_f32(const float* heads, int batch, int h, int w, float resize, float conf_thr, float* boxes,
                                         float* landms, float* keys, float* loc, float* conf, float* landm_raw, void* stream) {
    E4S_REQUIRE(heads && batch > 0 && h > 0 && w > 0, E4S_ERR_ARG);
    E4S_REQUIRE(h % 32 == 0 && w % 32 == 0, E4S_ERR_SHAPE);
    const int64_t priors = (int64_t)(h / 8) * (w / 8) * 2 * (1 + 4 + 16) / 16;
    E4S_REQUIRE(priors * batch < (1ll << 31), E4S_ERR_SHAPE);
    E4S_REQUIRE(!boxes || e4s_aligned16(boxes), E4S_ERR_ALIGN);
    const int64_t total = priors * batch;
    retina::decode_kernel<<<(unsigned)e4s_ceil_div(total, 256), 256, 0, (cudaStream_t)stream>>>(
        heads, batch, h, w, resize, conf_thr, boxes, landms, keys, loc, conf, landm_raw, (int)priors);
    return e4s_launch_status();
}

extern "C" int e4s_retinaface_nms_f32(const float* boxes, const float* landms, const float* keys, const int64_t* order, int batch,
                                      int num_priors, float conf_thr, float nms_thr, int top_k, int keep_top_k, float* dets,
                                      float* landms_out, int* count, void* stream) {
    E4S_REQUIRE(boxes && landms && keys && order && count && batch > 0 && num_priors > 0 && top_k >= 0 && keep_top_k >= 0,
                E4S_ERR_ARG);
    E4S_REQUIRE(keep_top_k == 0 || (dets && landms_out), E4S_ERR_ARG);
    E4S_REQUIRE(e4s_aligned16(boxes), E4S_ERR_ALIGN);
    const size_t smem = (size_t)(top_k < num_priors ? top_k : num_priors);
    E4S_REQUIRE(smem <= (size_t)e4s_smem_optin_limit() - 1024, E4S_ERR_SHAPE);
    static E4sSmemOptIn optin;
    if (const int rc = e4s_smem_optin(optin, retina::nms_kernel, smem)) return rc;
    retina::nms_kernel<<<batch, retina::NMS_THREADS, smem, (cudaStream_t)stream>>>(
        reinterpret_cast<const float4*>(boxes), landms, keys, order, num_priors, conf_thr, nms_thr, top_k, keep_top_k, dets,
        landms_out, count);
    return e4s_launch_status();
}
