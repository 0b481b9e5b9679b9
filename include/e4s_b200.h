/* e4s_b200 - C ABI of the CUDA-native (sm_90a, H100) E4S synthesis hot path.
 *
 * Drop-in boundary (SURVEY.md section 8b).  The reference binds its two native ops through
 * pybind11 modules JIT-built at import (src/models/stylegan2/op/upfirdn2d.py:8-14,
 * fused_act.py:9-15) and runs everything else through ATen/cuDNN.  This library replaces
 * that native layer: plain `extern "C"` functions over raw DEVICE pointers, int shapes and
 * a cudaStream_t (passed as void*).  Rules common to every entry point:
 *
 *   - returns 0 on success, a negative E4S_ERR_* code for a bad argument, or the positive
 *     cudaError_t of a failed launch; never throws, never allocates, never synchronises;
 *   - the caller owns every buffer and guarantees the layouts stated per function;
 *   - re-entrant; enqueues on `stream` of the CURRENT device and returns immediately;
 *   - all floating-point tensors are fp32, labels are uint8.
 *
 * Layout vocabulary: "planar" = [N, C, H, W] contiguous (the reference's NCHW);
 * "pixel-major" = [N, H, W, C] contiguous (torch channels_last storage of the same
 * logical NCHW tensor) - the layout the convolution kernels stream.
 */
#ifndef E4S_B200_H_
#define E4S_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define E4S_OK 0
#define E4S_ERR_ARG (-1)      /* null pointer / non-positive size */
#define E4S_ERR_SHAPE (-2)    /* unsupported shape (e.g. FIR larger than 8x8) */
#define E4S_ERR_ALIGN (-3)    /* pointer not aligned as the kernel requires */
#define E4S_ERR_NOT_ONEHOT (-4)
#define E4S_ERR_ARCH (-5)     /* device is not sm_90 */

/* Library version: major*10000 + minor*100 + patch. */
int e4s_version(void);
/* Static string naming the architecture the kernels were compiled for ("sm_90a"). */
const char* e4s_build_arch(void);
/* 0 if the current device can run this library (compute capability 9.0). */
int e4s_device_ok(void);

/* ---- upfirdn2d ---------------------------------------------------------------------
 * Replaces upfirdn2d_op / upfirdn2d_kernel, src/models/stylegan2/op/upfirdn2d_kernel.cu:52-272
 * (pybind surface upfirdn2d.cpp:12-23; Python semantics upfirdn2d.py:85-147).
 * x: planar [planes, in_h, in_w]; y: planar [planes, out_h, out_w];
 * fir: [kh, kw] row-major DEVICE pointer (kh, kw <= 8).  The op zero-stuffs by `up`, pads
 * (negative pad crops), applies a TRUE convolution (kernel flipped) and keeps every
 * `down`-th sample: out = (in*up + pad0 + pad1 - k)/down + 1, checked against out_h/out_w. */
int e4s_upfirdn2d_f32(const float* x, float* y, const float* fir, int planes, int in_h, int in_w,
                      int out_h, int out_w, int kh, int kw, int up_x, int up_y, int down_x, int down_y,
                      int pad_x0, int pad_x1, int pad_y0, int pad_y1, void* stream);

/* ---- fused bias + leaky ReLU -------------------------------------------------------
 * Replaces fused_bias_act_op / fused_bias_act_kernel, fused_bias_act_kernel.cu:18-99
 * (pybind fused_bias_act.cpp:11-21; Python fused_act.py:50-85), act=3 (lrelu).
 * Forward: y[i] = scale * lrelu(x[i] + bias[(i / step_b) % size_b], alpha); bias may be NULL.
 * Backward (grad=1): gx[i] = scale * (ref[i] > 0 ? g[i] : alpha * g[i]), ref = forward output. */
int e4s_bias_act_fwd_f32(const float* x, const float* bias, float* y, int64_t n, int step_b, int size_b,
                         float alpha, float scale, void* stream);
int e4s_bias_act_bwd_f32(const float* g, const float* ref, float* gx, int64_t n, float alpha, float scale,
                         void* stream);
/* Per-channel sum of gx over everything but the channel axis (grad of bias, fused_act.py:31-36).
 * gx viewed as [outer, size_b, step_b]; gb[size_b] is overwritten. */
int e4s_bias_grad_f32(const float* gx, float* gb, int64_t outer, int size_b, int step_b, void* stream);

/* ---- mask / index ops (bit-exact) ---------------------------------------------------
 * onehot [B, ncls, H, W] float -> label [B, H, W] uint8 (argmax).  *flag (device int, caller
 * zeroes it) is set to 1 if any pixel is not exactly one-hot (one 1.0, rest 0.0).
 * Replaces the float mask arithmetic of model.py:391-398 by an index map. */
int e4s_onehot_to_label_u8(const float* onehot, uint8_t* label, int* flag, int batch, int ncls, int h, int w,
                           void* stream);
/* label -> one-hot float, labelMap2OneHot, src/utils/torch_utils.py:166-172. */
int e4s_label_to_onehot_f32(const uint8_t* label, float* onehot, int batch, int ncls, int h, int w, void* stream);
/* Nearest resize of a label map with ATen's legacy 'nearest' index rule
 * (src = min(floor(dst * in/out), in-1), float32), as F.interpolate(mask, mode='nearest') does at
 * model.py:391,430 and psp_encoders.py:265. */
int e4s_label_resize_nearest_u8(const uint8_t* src, uint8_t* dst, int batch, int in_h, int in_w, int out_h,
                                int out_w, void* stream);
/* Class remap through a 256-entry LUT (device pointer); the CelebAMask-HQ 19->12 conversion of
 * src/datasets/dataset.py:153-209 is one such table. */
int e4s_label_remap_u8(const uint8_t* src, uint8_t* dst, const uint8_t* lut256, int64_t n, void* stream);
/* Shape swapping of the face-swapping pipeline (step 4 of scripts/face_swap.py:253): replaces
 * swap_head_mask_revisit_considerGlass, src/utils/swap_face_mask.py:33-83, a numpy routine on the host.
 * source / target: 12-class label maps (faceParser_label_list_detailed, :27-29) of n pixels each;
 * swapped: the recomposed label map; hole: 255 where no region claimed the pixel (filled with skin), else 0;
 * foreground (may be NULL): 1 where the swapped label is not background / hair / ear rings or the pixel is a hole
 * (scripts/face_swap.py:280-284), else 0.  hair_first selects :47-48 over :66-67. */
int e4s_swap_head_mask_u8(const uint8_t* source, const uint8_t* target, uint8_t* swapped, uint8_t* hole,
                          uint8_t* foreground, int64_t n, int hair_first, void* stream);
/* Flat (2*radius+1)^2 box dilation (erode = 0) or erosion (erode = 1) of uint8 masks [planes, h, w] with the
 * reference's 'geodesic' border (pixels outside the image are ignored): dilation / erosion of
 * src/utils/morphology.py:23-197 as scripts/face_swap.py:30-48 (create_masks) calls them.  radius <= 16;
 * src and dst must not alias. */
int e4s_mask_box_morph_u8(const uint8_t* src, uint8_t* dst, int planes, int h, int w, int radius, int erode,
                          void* stream);
/* The same on fp32 images (the reference's tensors are float): out-of-image positions count as -max_val (dilation)
 * or +max_val (erosion), exactly the padding of morphology.py:83-86, 170-173 (default max_val 1e4). */
int e4s_box_morph_f32(const float* src, float* dst, int planes, int h, int w, int radius, int erode, float max_val,
                      void* stream);
/* Region mean pooling, FSEncoder_PSP.get_per_comp_styleCode, psp_encoders.py:264-283.
 * feats: pixel-major [B, H, W, C]; label: [B, H, W] uint8 (already at feature resolution), ncls <= 64 (labels >= ncls
 * are ignored);
 * out: [B, ncls, C] (zero for empty regions); area: [B, ncls] int32 scratch/outputs. */
int e4s_region_mean_f32(const float* feats, const uint8_t* label, float* out, int* area, int batch, int ncls,
                        int h, int w, int c, void* stream);

/* ---- modulated convolution ----------------------------------------------------------
 * Demodulation coefficients, model.py:279-281 in the shared-weight form of model.py:245-274:
 * demod[r, o] = rsqrt(sum_i s[r,i]^2 * wsq[o,i] + eps), wsq[o,i] = sum_k (scale*W[o,i,k])^2.
 * s: [rows, cin], wsq: [cout, cin], demod: [rows, cout]. */
int e4s_demod_f32(const float* s, const float* wsq, float* demod, int rows, int cin, int cout, float eps,
                  void* stream);
/* The same on the tiled small-GEMM kernel (csrc/linear.cu; cin % 4 == 0, cout % 4 == 0): what the generator uses. */
int e4s_demod_gemm_f32(const float* s, const float* wsq, float* demod, int rows, int cin, int cout, float eps, float* workspace,
                       void* stream);

/* Many independent small fp32 products in ONE launch (csrc/linear.cu): the 26 EqualLinear style modulations of a synthesis
 * forward (model.py:276, one per ModulatedConv2d) as one call, the 17 demodulation products (model.py:279-281) as a second.
 *   rsqrt_eps <  0:  y = x w^T + bias            x: [m, k] rows ldx floats apart (a latent slice is read in place),
 *   rsqrt_eps >= 0:  y = rsqrt((x*x) w^T + eps)  w: [n, k] (nn.Linear layout), bias: [n] | NULL, y: [m, n] contiguous.
 * n, k, ldx multiples of 4; pointers 16-byte aligned.  `problems` is a HOST array of device pointers (copied into kernel
 * parameters, E4S_LINEAR_MULTI_MAX per launch); K is never split, so the result is deterministic and needs no workspace. */
typedef struct E4sLinearProblem {
    const float* x;
    const float* w;
    const float* bias;
    float* y;
    int m, n, k, ldx;
    float rsqrt_eps;
    int reserved;
} E4sLinearProblem;
#define E4S_LINEAR_MULTI_MAX 48
int e4s_linear_multi_f32(const E4sLinearProblem* problems, int nproblems, void* stream);

/* Region-selected modulated 3x3 convolution with fused noise + bias + leaky-ReLU epilogue:
 * one call = one StyledConv.forward (model.py:382-406) for every region at once.
 *
 *   y[b,p,o] = act( demod[b,c(p),o] * sum_{i,k} wt[ph(p)][k][i][o] * s[b,c(p),i] * x[b,p+k,i]
 *                   + noise_w * noise[b,p] + bias[o] )
 *
 * x: pixel-major [B, H, W, Cin].  y: pixel-major [B, Ho, Wo, Cout] with Ho = H*(up?2:1).
 * s: [B, ncls, Cin] post-EqualLinear styles (model.py:276); demod: [B, ncls, Cout] or NULL (no
 * demodulation).  label: [B, Ho, Wo] uint8 class of every OUTPUT pixel, or NULL when ncls == 1
 * (unmasked layer).  wt: prepared weights [nphase, 9, Cin, Cout], already multiplied by
 * 1/sqrt(9*Cin); nphase = 1 for the plain conv, 4 for the up-sampling layer where the stride-2
 * transposed conv and the [1,3,3,1] blur (model.py:287-300) are folded into one 3x3 kernel per
 * output parity (see DESIGN.md).  noise: [noise_b, Ho, Wo] with noise_b in {1, B}, or NULL;
 * noise_w: DEVICE pointer to the scalar NoiseInjection.weight; bias: [Cout] or NULL.
 * act != 0 applies sqrt(2)*lrelu(.,0.2) (FusedLeakyReLU, fused_act.py:72-85). */
int e4s_modconv3x3_fwd_f32(const float* x, const float* wt, const float* s, const float* demod,
                           const uint8_t* label, const float* noise, const float* noise_w, const float* bias,
                           float* y, int batch, int h, int w, int cin, int cout, int ncls, int up, int noise_b,
                           int act, void* stream);

/* Tensor-core (mma.sync bf16) implementation of the same contract as e4s_modconv3x3_fwd_f32 for cin % 32 == 0 and
 * cout % 32 == 0 (csrc/wgmma_conv_rs.cu; up = 1: csrc/wgmma_conv_smem.cu).  Weights arrive pre-split into bf16 planes
 * w_hilo_bf16 = [2 (hi, lo)][nphase][9][Cout][Cin] with w = hi + lo to ~2^-17 relative (prepared once); activations
 * are split on the fly, three bf16 MMAs per product accumulate in fp32 registers (error ~1e-5 relative to fp32).  One
 * pass per tile whatever the number of regions in it. */
int e4s_modconv3x3_tcr_fwd(const float* x, const void* w_hilo_bf16, const float* s, const float* demod,
                           const uint8_t* label, const float* noise, const float* noise_w, const float* bias,
                           float* y, int batch, int h, int w, int cin, int cout, int ncls, int up, int noise_b,
                           int act, void* stream);
/* The same contract for an UNMASKED up-sampling layer (label NULL, ncls == 1; model.py:287-300 with one style per sample),
 * computed as the stride-2 transposed convolution followed by the blur instead of four folded parity kernels: 9 instead of
 * 36 multiply-accumulates per input pixel and channel pair.  Two launches (csrc/wgmma_convt.cu):
 *   1. a tensor-core GEMM writes the raw transposed-convolution output space-to-depth into
 *      t_buf [B, H+1, W+1, 4*Cout] (channel (a, c, o) = output pixel (2m+a, 2n+c)); no demodulation, noise, bias or act;
 *   2. a streaming pass applies the 4x4 FIR (true convolution, pad 1, as upfirdn2d) and the epilogue of
 *      e4s_modconv3x3_fwd_f32 (demod, noise, bias, act) into y [B, 2H, 2W, Cout].
 * wt_hilo_bf16: [2 (hi, lo)][1][9][4*Cout][Cin], rows (a, c, o): the weight tap (ky, kx) that parity (a, c) takes from source
 * pixel (m-1+dy, n-1+dx) at 3x3 tap index 3 dy + dx (dy, dx in {0, 1}; a = 0: dy = 1 -> ky = 0, dy = 0 -> ky = 2;
 * a = 1: dy = 1 -> ky = 1, dy = 0 zero; the same along x), zero elsewhere; already multiplied by 1/sqrt(9*Cin).
 * fir4x4: the layer's blur FIR (already scaled by 4, model.py:34-53), DEVICE pointer.  s: [B, 1, Cin]; demod: [B, 1, Cout]
 * or NULL.  t_buf is scratch owned by the caller and overwritten.  cin % 32 == 0, cout % 32 == 0.  Bit reproducible. */
int e4s_modconv3x3_up_tcr_fwd(const float* x, const void* wt_hilo_bf16, const float* fir4x4, const float* s,
                              const float* demod, const float* noise, const float* noise_w, const float* bias,
                              float* t_buf, float* y, int batch, int h, int w, int cin, int cout, int noise_b, int act,
                              void* stream);
/* The same contract for a MASKED up-sampling layer (label [B, 2H, 2W], s [B, ncls, Cin], demod [B, ncls, Cout] or NULL):
 * through the blur, T' pixel (m, n) reaches only the output pixels of its 5 x 5 window [2m-2, 2m+2] x [2n-2, 2n+2], so it is
 * computed once per region present there.  Four launches (csrc/wgmma_convt.cu, the fallback in csrc/wgmma_conv_smem.cu):
 *   1. per sample, the row list over the (H+1) x (W+1) T' pixels: need [B, H+1, W+1] the region bitmask of the window,
 *      base [B, H+1, W+1] the exclusive prefix sum of its popcount, count [B] the total (past cap the count stops
 *      early: only count > cap is meaningful), rows [B, cap] the packed
 *      (m << 18 | n << 5 | region) of each row;
 *   2. the tensor-core GEMM of e4s_modconv3x3_up_tcr_fwd over those rows, each row's operand scaled by its region's style,
 *      into t_buf [B, cap, 4*Cout];
 *   3. the blur pass: output pixel (Y, X) of region r reads T' row base + popcount(need & ((1 << r) - 1)) at each of
 *      its 4 x 4 taps, then the epilogue with demod[b, r];
 *   4. the folded parity kernel of e4s_modconv3x3_tcr_fwd (w_hilo_bf16) for the samples with count > cap; 2 - 3 skip
 *      those samples.  No host decision: the launches are the same for any label map (CUDA-graph capturable).
 * need, base, count, rows and t_buf are scratch owned by the caller.  h + 1 < 16384, w + 1 < 8192.  Bit reproducible. */
int e4s_modconv3x3_up_masked_tcr_fwd(const float* x, const void* wt_hilo_bf16, const void* w_hilo_bf16, const float* fir4x4,
                                     const float* s, const float* demod, const uint8_t* label, const float* noise,
                                     const float* noise_w, const float* bias, uint32_t* need, int* base, int* count,
                                     uint32_t* rows, float* t_buf, float* y, int batch, int h, int w, int cin, int cout,
                                     int ncls, int cap, int noise_b, int act, void* stream);
/* Bit reproducibility of the tensor-core convolutions (forward kernels).  The forward kernels accumulate every output in a
 * fixed order, so their results are bit reproducible with either setting.  The initial value comes from the environment
 * variable E4S_B200_DETERMINISTIC.  e4s_get_deterministic returns the current setting (0 / 1). */
int e4s_set_deterministic(int on);
int e4s_get_deterministic(void);

/* ---- RGI encoder conv stack (src/models/encoders/helpers.py:122-144, psp_encoders.py:285-309) ------------------
 * Plain 3x3 convolution, padding 1, on the tensor-core kernel.
 * x: pixel-major [B, H, W, Cin]; w_hilo_bf16: [2][1][9][Cout][Cin]; scale/shift: optional per-(sample, channel)
 * affine [B, Cin] applied to in-image pixels while staging (InstanceNorm folded onto the operand; zero padding
 * stays zero); prelu_slope: optional [Cout] PReLU epilogue.
 * out_stride 1: y [B, H, W, Cout].  2: every pixel is computed, the even ones are stored, y [B, H/2, W/2, Cout].
 * 4: space-to-depth store, y [B, H/2, W/2, 4 Cout] with channel (y & 1, x & 1, c) - what the NEXT layer wants when it is a
 *    stride-2 convolution (helpers.py:138: conv2 of the first unit of a stage): on that tensor the stride-2 kernel is a
 *    stride-1 kernel over 4 Cin channels of which only the taps (dy, dx) in {-1, 0}^2 are non-zero.
 * tap_mask: bit t (row-major 3x3) set = tap t is multiplied, 0 = all nine; masked taps are neither loaded nor issued
 *    (their weights must be zero for the result to be the full convolution).  0x1B = the four taps of the case above. */
int e4s_conv3x3_tcr_f32(const float* x, const void* w_hilo_bf16, const float* scale, const float* shift,
                        const float* prelu_slope, float* y, int batch, int h, int w, int cin, int cout, int out_stride,
                        int tap_mask, void* stream);
/* e4s_conv3x3_tcr_f32 (same operand affine, out_stride, tap_mask and mainloop) with the epilogue
 * y = relu?(acc + bias[o] + residual): bias [Cout] or NULL; residual laid out like y (pixel-major for out_stride 1) or NULL;
 * relu != 0 applies ReLU.  The BiSeNet parser's convolutions: BatchNorm folded into the weights and bias, the residual add of
 * a BasicBlock, the ReLU. */
int e4s_conv3x3_bias_tcr_f32(const float* x, const void* w_hilo_bf16, const float* scale, const float* shift,
                             const float* bias, const float* residual, float* y, int batch, int h, int w, int cin, int cout,
                             int out_stride, int tap_mask, int relu, void* stream);

/* ---- RealESRNet x4 (src/pretrained/gpen/sr_model/rrdbnet_arch.py: RRDBNet, num_feat 32, num_grow_ch 32) -------------
 * Plain 3x3 convolution, padding 1, on the tensor-core kernel, over pixel-PITCHED operands: x [B, H, W, *] with pixel
 * stride x_ld >= cin floats, y [B, Ho, Wo, *] with pixel stride y_ld >= cout floats (both multiples of 4); x and y may be
 * channel slices of wider buffers, passed as channel-offset pointers (16-byte aligned), and may lie in the same buffer when
 * the channel ranges read and written do not overlap - a residual dense block keeps x, x1 .. x4 in one [B, H, W, 160]
 * buffer, conv k reading channels [0, 32 k) and writing [32 k, 32 k + 32).  w_hilo_bf16: [2][1][9][Cout][Cin] as
 * e4s_conv3x3_tcr_f32.  up != 0: nearest 2x up-sampling of x first (x is [B, H, W], y [B, 2H, 2W]; the up-sampled tensor is
 * never written), else y is [B, H, W].  Epilogue, in the reference modules' order of operations:
 *   t = (acc + bias[o]) * alpha;  t += r0 (if given);  t = t * beta + r1 (if given);  y = t > 0 ? t : t * lrelu_slope
 * with bias [Cout] or NULL, r0 / r1 pitched like y (y_ld) or NULL, lrelu_slope 1 for no activation.  A residual may be the
 * element it is stored over (each element is read by the thread that writes it). */
int e4s_conv3x3_dense_tcr_f32(const float* x, int x_ld, const void* w_hilo_bf16, const float* bias, float alpha, const float* r0,
                              float beta, const float* r1, float* y, int y_ld, int batch, int h, int w, int cin, int cout, int up,
                              float lrelu_slope, void* stream);
/* The RGB-side 3x3 convolutions of RRDBNet (padding 1, + bias, fp32 on CUDA cores), w3x3 [Cout][Cin][3][3] (nn.Conv2d),
 * bias [Cout].  cin 3, cout 32 (conv_first): x planar [B, 3, H, W], y pixel-major with pitch y_ld (x_ld unused).
 * cin 32, cout 3 (conv_last): x pixel-major with pitch x_ld, y planar [B, 3, H, W] (y_ld unused).  Other shapes: E4S_ERR_SHAPE. */
int e4s_conv3x3_rgb_f32(const float* x, int x_ld, const float* w3x3, const float* bias, float* y, int y_ld, int batch, int h,
                        int w, int cin, int cout, void* stream);

/* ---- GPEN's ParseNet (src/pretrained/gpen/face_parse/parse_model.py; FaceParse's configuration, 512 x 512) -----------
 * e4s_conv3x3_dense_tcr_f32 (same operands, pitches, weights and epilogue) with REFLECTION padding 1 (nn.ReflectionPad2d
 * before the convolution) in place of zero padding.  h, w: the grid of x, both >= 2.  mode:
 *   0: stride 1, y [B, h, w]: halo row -1 reads row 1, row h reads row h - 2 (the same for columns);
 *   1: nearest 2x up-sampling first, y [B, 2h, 2w]: reflection padding of the up-sampled grid equals replicate padding of x;
 *   2: stride 2 over the space-to-depth operand: x [B, h, w, cin] is e4s_space_to_depth_f32's output of a [B, 2h, 2w, cin / 4]
 *      tensor, w_hilo_bf16 holds only the taps (dy, dx) in {-1, 0}^2 (as e4s_conv3x3_tcr_f32 with tap_mask 0x1B), y [B, h, w]:
 *      reflection padding 1 of the 2h x 2w input then equals row and column -1 of x replicating row and column 0 (no padding
 *      is read at the bottom or right).
 * Other modes: E4S_ERR_ARG.  Bit reproducible. */
int e4s_conv3x3_reflect_tcr_f32(const float* x, int x_ld, const void* w_hilo_bf16, const float* bias, float alpha,
                                const float* r0, float beta, const float* r1, float* y, int y_ld, int batch, int h, int w, int cin,
                                int cout, int mode, float lrelu_slope, void* stream);
/* The RGB-side 3x3 convolutions of ParseNet (reflection padding 1, + bias, fp32 on CUDA cores), w3x3 [Cout][Cin][3][3],
 * bias [Cout]; h, w >= 2: the network's grid.
 * cin 3, cout 64 (encoder.0): y pixel-major [B, h, w, *] with pitch y_ld (multiple of 4).  prep 0: x planar [B, 3, h, w]
 *   (hs = h, ws = w).  prep 1: x planar BGR [B, 3, hs, ws] and the network input is F.interpolate(x.flip(1) * 2 - 1, (h, w))
 *   (mode 'nearest', the same fp32 arithmetic), read as the pixels are loaded.
 * cin 64, cout 3 (out_img_conv): x pixel-major with pitch x_ld, y planar [B, 3, h, w]; prep must be 0.
 * Other shapes: E4S_ERR_SHAPE.  Each output sums taps row-major, channels ascending, then adds the bias. */
int e4s_conv3x3_rgb_reflect_f32(const float* x, int x_ld, int hs, int ws, int prep, const float* w3x3, const float* bias,
                                float* y, int y_ld, int batch, int h, int w, int cin, int cout, void* stream);
/* ParseNet's mask head: out_mask_conv (cin 64 -> ncls 19, 3x3, reflection padding 1, + bias) over x pixel-major [B, h, w, *]
 * (pitch x_ld), then per pixel the first-index argmax k over the 19 logits and lut[k] (uint8 [19], on the device:
 * FaceParse.MASK_COLORMAP).  Outputs, each optional (at least one): logits planar [B, 19, h, w]; mask_u8 [B, h, w];
 * mask_i64 [B, h, w] (int64, the dtype of FaceParse.process_tensor).  No logits need be written for the masks. */
int e4s_gpen_parse_head_u8(const float* x, int x_ld, const float* w3x3, const float* bias, const uint8_t* lut, float* logits,
                           uint8_t* mask_u8, int64_t* mask_i64, int batch, int h, int w, int cin, int ncls, void* stream);

/* ---- GPEN's RetinaFace-R50 detector (src/pretrained/gpen/face_detect/; cfg_re50, phase 'test') ------------------------
 * e4s_conv3x3_dense_tcr_f32 (same operands, pitches, weights layout, epilogue; zero padding 1, no up-sampling) with the N tile
 * chosen from cout alone, so that a sample's output is bit identical whatever the batch.  stride 1: x [B, h, w, cin] ->
 * y [B, h, w].  stride 2: x [B, h, w, cin] is e4s_space_to_depth_f32's output of a [B, 2h, 2w, cin / 4] tensor and
 * w_hilo_bf16 holds only the taps (dy, dx) in {-1, 0}^2 (as e4s_conv3x3_tcr_f32 with tap_mask 0x1B), y [B, h, w].  Other
 * strides: E4S_ERR_ARG.  The detector's 3x3 convolutions. */
int e4s_conv3x3_zero_tcr_f32(const float* x, int x_ld, const void* w_hilo_bf16, const float* bias, float alpha, const float* r0,
                             float beta, const float* r1, float* y, int y_ld, int batch, int h, int w, int cin, int cout,
                             int stride, float lrelu_slope, void* stream);
/* 1x1 convolution on the tensor-core kernel's plain mode, pointwise: y [B, h, w, *] (pixel pitch y_ld) from x
 * [B, stride h, stride w, *] (pitch x_ld) read at (stride y, stride x), stride 1 or 2 (a strided shortcut needs no
 * space-to-depth pass).  w_hilo_bf16: [2][Cout][Cin] (bf16 hi, lo planes of the weight).  cin, cout multiples of 32; pitches
 * multiples of 4 floats; pointers 16-byte aligned.  Epilogue, in this order:
 *   t = (acc + bias[o]) * alpha;  t += r0 (if given, pitched like y);  t = t > 0 ? t : t * lrelu_slope;  t += r_up (if given)
 * with r_up [B, h / 2, w / 2, *] (pitch r_up_ld, h and w even) read at (y >> 1, x >> 1): FPN's lateral plus the nearest-2x
 * up-sampled coarser level.  r0 is a bottleneck's residual (before its ReLU).  Each output's sum order is fixed: bit
 * reproducible and independent of the batch. */
int e4s_conv1x1_tcr_f32(const float* x, int x_ld, const void* w_hilo_bf16, const float* bias, float alpha, const float* r0,
                        const float* r_up, int r_up_ld, float* y, int y_ld, int batch, int h, int w, int cin, int cout, int stride,
                        float lrelu_slope, void* stream);
/* 3x3x3 convolution (padding 1) on the tensor-core kernel's plain mode: face-vid2vid's UpBlock3d and keypoint head.
 * x [B, h, w, D, cin] -> y [B, ho, wo, D, cout] (ho, wo = h, w, or 2h, 2w when up != 0: nearest up-sampling by (1, 2, 2)
 * first), y = relu?(acc + bias[o]).  w_hilo_bf16: [2][9][Cout][3 Cin], element (hl, 3 ky + kx, o, kz Cin + c) of the
 * Conv3d weight [Cout, Cin, kz, ky, kx] split into bf16 hi, lo planes.  cin, cout multiples of 32; pointers 16-byte
 * aligned.  The B D depth slices are tiled as a mosaic (e4s_conv3d_tcr_plan): small slices share pixel tiles, separated
 * by zero gutters.  Each output's sum order is fixed: bit reproducible and independent of the batch. */
int e4s_conv3d_tcr_f32(const float* x, const void* w_hilo_bf16, const float* bias, float* y, int batch, int depth, int h, int w,
                       int cin, int cout, int up, int relu, void* stream);
/* e4s_conv3d_tcr_f32 over channel slices: x [B, h, w, D, *] with voxel pitch x_vp (floats, >= cin), y [B, ho, wo, D, *]
 * with voxel pitch y_vp (>= cout), each a channel range of a wider contiguous buffer (face-vid2vid's dense-motion
 * hourglass keeps each skip concatenation in one buffer whose producers write disjoint channel ranges of it).  Pitches
 * multiples of 4; otherwise as e4s_conv3d_tcr_f32, with the same results at the same sum order. */
int e4s_conv3d_pitched_tcr_f32(const float* x, int x_vp, const void* w_hilo_bf16, const float* bias, float* y, int y_vp, int batch,
                               int depth, int h, int w, int cin, int cout, int up, int relu, void* stream);
/* e4s_conv3d_tcr_f32 (no up-sampling) with a residual added after the bias, before the ReLU: y = relu?(acc + bias +
 * residual), residual contiguous [B, h, w, D, cout] (face-vid2vid's ResBlock3d: conv2 + x). */
int e4s_conv3d_residual_tcr_f32(const float* x, const void* w_hilo_bf16, const float* bias, const float* residual, float* y,
                                int batch, int depth, int h, int w, int cin, int cout, int relu, void* stream);

/* ---- face-vid2vid's occlusion-aware SPADE generator (src/pretrained/face_vid2vid/modules/generator.py, vox-256.yaml) ----
 * e4s_conv3x3_zero_tcr_f32 over the nearest up-sampling of x [B, h, w, cin] (pitch x_ld) by 2^up_shift (1 or 2), read
 * through the halo copy: y [B, h 2^up_shift, w 2^up_shift, cout] (pitch y_ld) = lrelu_slope(acc + bias).  The N tile
 * follows cout only: bit identical at any batch.  The SPADE blocks' mlp_shared at 128^2 and 256^2 from the 64^2 map. */
int e4s_conv3x3_zero_up_tcr_f32(const float* x, int x_ld, const void* w_hilo_bf16, const float* bias, float* y, int y_ld, int batch,
                                int h, int w, int cin, int cout, int up_shift, float lrelu_slope, void* stream);
/* SPADE: the 3x3 (zero padding 1) gamma / beta convolutions of actv [B, h, w, cin] (pitch actv_ld) as one GEMM of 2 c
 * interleaved columns (w_hilo_bf16 [2][1][9][2 c][cin], row 2 k gamma k, row 2 k + 1 beta k; bias [2 c] likewise), whose
 * epilogue writes y [B, h, w, c] (pitch y_ld) = lrelu_slope((x scale + shift) (1 + gamma) + beta): x [B, h, w, c]
 * (pitch x_ld; x_half 1: [B, h / 2, w / 2, c] read at (y >> 1, x >> 1), the nearest up-sampling of x), scale / shift
 * [B, c] its instance-norm statistics (e4s_instnorm_stats_fixed_f32).  Neither the normalised x nor gamma / beta is
 * written.  The N tile follows c only: bit identical at any batch. */
int e4s_spade_tcr_f32(const float* actv, int actv_ld, const void* w_hilo_bf16, const float* bias, const float* x, int x_ld,
                      int x_half, const float* scale, const float* shift, float* y, int y_ld, int batch, int h, int w, int cin,
                      int c, float lrelu_slope, void* stream);
/* e4s_conv1x1_tcr_f32 (stride 1, no residuals) times a per-pixel factor: y = (acc + bias) factor[b, y, x], factor
 * contiguous [B, h, w] (the generator's fourth convolution times the occlusion map). */
int e4s_conv1x1_factor_tcr_f32(const float* x, int x_ld, const void* w_hilo_bf16, const float* bias, const float* factor, float* y,
                               int y_ld, int batch, int h, int w, int cin, int cout, void* stream);
/* deform_input: F.grid_sample (trilinear, zero padding, align_corners=False) of vol [B, h, w, d, 32] at deformation
 * [B, d, h, w, 3] -> y [B, h, w, d 32], channel z 32 + c (contiguous). */
int e4s_vid2vid_warp_f32(const float* vol, const float* deformation, float* y, int batch, int d, int h, int w, void* stream);
/* e4s_conv3x3_rgb_f32's kernel with an activation after the bias: cin 3 -> cout 64 with act 1 (ReLU; planar x, pixel-
 * pitched y), cin 64 -> cout 3 with act 2 (sigmoid; pixel-pitched x, planar y). */
int e4s_conv3x3_rgb_act_f32(const float* x, int x_ld, const float* w3x3, const float* bias, float* y, int y_ld, int batch, int h,
                            int w, int cin, int cout, int act, void* stream);
/* 7x7 convolution (zero padding 3) of every depth slice of x [B, h, w, D, cin] -> y [B, D, h, w, 128]:
 * y[b, z, y, x, n] = sum over (ky, kx, c) of w[ky 7 + kx][n][c] x[b, y + ky - 3, x + kx - 3, z, c].  w_hilo_bf16:
 * [2][49][128][cin] bf16 hi, lo planes.  cin a multiple of 32, h of 8, w of 16; pointers 16-byte aligned.  face-vid2vid's
 * dense-motion mask (7x7x7) and occlusion (7x7 over the c D + d channels) as one GEMM per slice, combined over the depths
 * by e4s_vid2vid_motion_combine_f32.  Each output's sum order is fixed: bit reproducible and independent of the batch. */
int e4s_conv7x7_slices_tcr_f32(const float* x, const void* w_hilo_bf16, float* y, int batch, int depth, int h, int w, int cin,
                               void* stream);
/* The mosaic e4s_conv3d_tcr_f32 tiles for an output of B x D slices of ho x wo: mosaic_h x mosaic_w pixels, covered by
 * ceil(mosaic_h / 8) x ceil(mosaic_w / 16) tiles of 128 pixel rows. */
int e4s_conv3d_tcr_plan(int batch, int depth, int ho, int wo, int* mosaic_h, int* mosaic_w);
/* face-vid2vid KPDetector input prep (AntiAliasInterpolation2d, scale 1/4): x planar [B, 3, h, w] (h, w multiples of 4),
 * filter [3, 13, 13] (the loaded `down.weight`) -> y pixel-major [B, h / 4, w / 4, 32]: channel c < 3 the zero-padded
 * (6) depthwise filter at (4 y, 4 x), channels 3..31 zero. */
int e4s_vid2vid_kp_prep_f32(const float* x, const float* filter, float* y, int batch, int h, int w, void* stream);
/* AvgPool2d(2) of pixel-major [B, h, w, c] (h, w even, c a multiple of 4) -> [B, h / 2, w / 2, c]. */
int e4s_avgpool2_f32(const float* x, float* y, int batch, int h, int w, int c, void* stream);
/* AvgPool3d((1, 2, 2)) of contiguous x [B, h, w, d, c] (h, w even, c a multiple of 4) -> y [B, h / 2, w / 2, d, *] at voxel
 * pitch y_vp (>= c, a multiple of 4): a channel slice of a wider buffer. */
int e4s_avgpool2_vox_f32(const float* x, float* y, int y_vp, int batch, int h, int w, int d, int c, void* stream);
/* face-vid2vid DenseMotionNetwork (vox-256.yaml: 15 keypoints, compress 4, feature_channel 32).
 * Compress: x NCDHW [B, 32, d, h, w], wb [4 x 32 weights (BatchNorm folded), 4 biases] -> y [B, d, h, w, 4] =
 * relu(bias + w x), channels in order. */
int e4s_vid2vid_compress_f32(const float* x, const float* wb, float* y, int batch, int d, int h, int w, void* stream);
/* Hourglass input: comp [B, d, h, w, 4] (e4s_vid2vid_compress_f32), kp_driving, kp_source [B, 15, 3] -> y [B, h, w, d, *]
 * (voxel pitch y_vp >= 96, a multiple of 4): channel 5 k + j of voxel (y, x, z), k = 0 .. 15, is for j = 0 the heatmap
 * difference exp(-50 |g - kp_driving[k - 1]|^2) - exp(-50 |g - kp_source[k - 1]|^2) (0 for k = 0) and for j = 1 .. 4 the
 * trilinear sample (F.grid_sample, align_corners=False, zero padding) of comp channel j - 1 at the sparse motion: g for
 * k = 0, else (g - kp_driving[k - 1]) + kp_source[k - 1], with g = make_coordinate_grid's (x, y, z); channels 80..95
 * zero. */
int e4s_vid2vid_motion_input_f32(const float* comp, const float* kp_driving, const float* kp_source, float* y, int y_vp, int batch,
                                 int d, int h, int w, void* stream);
/* Mask and occlusion from p [B, d, h, w, 128] (e4s_conv7x7_slices_tcr_f32 with columns 16 dz + o = the mask weights of
 * kernel depth dz, 112 + d' = the occlusion weights of input depth d'; d <= 16): logits[z, o] = (sum over dz of p[z + dz - 3,
 * 16 dz + o], depths outside skipped) + mask_bias[o]; mask [B, 16, d, h, w] = softmax over o; deformation [B, d, h, w, 3]
 * = sum over k of mask[k] * (the sparse motion k of e4s_vid2vid_motion_input_f32); occlusion [B, 1, h, w] =
 * sigmoid((sum over d' of p[d', 112 + d']) + occ_bias[0]). */
int e4s_vid2vid_motion_combine_f32(const float* p, const float* mask_bias, const float* occ_bias, const float* kp_driving,
                                   const float* kp_source, float* mask, float* deformation, float* occlusion, int batch, int d,
                                   int h, int w, void* stream);
/* face-vid2vid keypoint heatmaps: logits [B, h, w, d, ld] (keypoint k at channel k < num_kp <= ld) -> kp [B, num_kp, 3],
 * per keypoint softmax(logits / temperature) over the d h w voxels and the expectation of (x, y, z), each 2 i / (n - 1) - 1
 * along W, H, D.  Fixed summation order: bit reproducible and independent of the batch. */
int e4s_vid2vid_heatmap_f32(const float* logits, int ld, float temperature, float* kp, int batch, int num_kp, int d, int h,
                            int w, void* stream);
/* Detector input: x planar BGR [B, 3, h, w], uint8 (x_u8 != 0) or fp32 pixel values -> y planar fp32 x - (104, 117, 123). */
int e4s_retinaface_prep_f32(const void* x, int x_u8, float* y, int batch, int h, int w, void* stream);
/* Per prior of an h x w image (multiples of 32; P = 2 (h w / 64 + h w / 256 + h w / 1024) priors in the reference's order:
 * level (steps 8, 16, 32), row, column, anchor): heads holds the three levels' head outputs one after another, level l as
 * pixel-major [B, h / s_l, w / s_l, 32] with channels class 4 | bbox 8 | landmark 20 (anchor a: class 2a.., bbox 4 + 4a..,
 * landmark 12 + 10a..).  PriorBox's anchor is computed in double and rounded to float.  Outputs, each optional:
 *   loc [B, P, 4], conf [B, P, 2] (softmax), landm_raw [B, P, 10]: RetinaFace.forward's outputs;
 *   boxes [B, P, 4] (16-byte aligned) = decode(loc) * [w, h, w, h] / resize, landms [B, P, 10] = decode_landm * [w, h, ...] /
 *   resize, both in box_utils' fp32 operation order; keys [B, P] = the face score where it is > conf_thr, else -inf. */
int e4s_retinaface_decode_f32(const float* heads, int batch, int h, int w, float resize, float conf_thr, float* boxes,
                              float* landms, float* keys, float* loc, float* conf, float* landm_raw, void* stream);
/* Selection and greedy NMS, one CTA per image.  keys [B, P] sorted descending with ties in ascending prior index (a stable
 * sort of the decode's keys), order [B, P] int64 the prior of each sorted entry, boxes [B, P, 4] / landms [B, P, 10] the
 * decode's.  Candidates: the first min(top_k, P) entries with key > conf_thr.  NMS in py_cpu_nms's fp32 arithmetic: a
 * candidate is dropped when its overlap with a kept box is not <= nms_thr (NaN drops).  Writes count[b] <= keep_top_k and
 * dets [B, keep_top_k, 5] (x1, y1, x2, y2, score) / landms_out [B, keep_top_k, 10] (x1..x5, y1..y5) in kept order; slots past
 * count are untouched.  min(top_k, P) bytes of shared memory per CTA. */
int e4s_retinaface_nms_f32(const float* boxes, const float* landms, const float* keys, const int64_t* order, int batch,
                           int num_priors, float conf_thr, float nms_thr, int top_k, int keep_top_k, float* dets, float* landms_out,
                           int* count, void* stream);

/* InstanceNorm2d statistics (biased variance, eps) of a pixel-major tensor as an affine: scale = rstd,
 * shift = -mean*rstd, both [B, C].  sums_ws: [B, C, 2] workspace. */
int e4s_instnorm_affine_f32(const float* x, float* sums_ws, float* scale, float* shift, int batch, int h, int w, int c,
                            float eps, void* stream);
/* InstanceNorm2d statistics (biased variance) of x [B, h, w, c] (pixel pitch x_ld) as scale = 1 / sqrt(var + eps),
 * shift = -mean scale, each [B, c], summed in double in an order fixed by h, w and c (no atomics): bit identical at any
 * batch.  part_ws: [B, ceil(h w / 1024), c, 2] doubles of workspace. */
int e4s_instnorm_stats_fixed_f32(const float* x, int x_ld, double* part_ws, float* scale, float* shift, int batch, int h, int w,
                                 int c, float eps, void* stream);
/* out = act(alpha * (y*y_scale + y_shift) + shortcut), shortcut = shortcut[b, sc_stride*p, c] (* sc_scale + sc_shift
 * when given); act = PReLU(prelu_slope) when given.  One residual-unit tail of bottleneck_IR_SE_Ours. */
int e4s_norm_residual_f32(const float* y, const float* y_scale, const float* y_shift, float alpha, const float* shortcut,
                          const float* sc_scale, const float* sc_shift, int sc_stride, const float* prelu_slope, float* out,
                          int batch, int h, int w, int c, void* stream);

/* Region-selected 1x1 modulated conv to RGB + bias + up-sampled skip: one ToRGB.forward
 * (model.py:422-448).  x: pixel-major [B, H, W, Cin]; wrgb: [3, Cin] (already scaled by
 * 1/sqrt(Cin)); s: [B, ncls, Cin]; label: [B, H, W] or NULL (ncls==1); bias: [3];
 * skip: planar [B, 3, H/2, W/2] or NULL; fir4x4: the Upsample FIR (model.py:34-53), DEVICE pointer,
 * may be NULL when skip is NULL; out: planar [B, 3, H, W]. */
int e4s_torgb_fwd_f32(const float* x, const float* wrgb, const float* s, const uint8_t* label,
                      const float* bias, const float* skip, const float* fir4x4, float* out, int batch, int h,
                      int w, int cin, int ncls, void* stream);

/* ---- backward (first order; generator weights are frozen, networks.py:69-71) -----------------
 * Input- and style-gradient of e4s_modconv3x3_fwd_f32 (replaces autograd through F.conv2d/conv_transpose2d with
 * per-sample weights, model.py:277-316, i.e. one cuDNN dgrad + wgrad per region per layer in the reference).
 * gy, y: pixel-major [B, Ho, Wo, Cout] (y = forward output, needed when act != 0); x: forward input;
 * wd: [nphase, 9, Cout, Cin] = forward weights with taps flipped and channels transposed; gx [B, H, W, Cin] is
 * overwritten (may be NULL); gs [B, ncls, Cin] receives the CONV-PATH style gradient by atomic accumulation
 * (caller zeroes it; may be NULL).  The demodulation-path term is assembled from e4s_class_reduce_f32. */
int e4s_modconv3x3_bwd_f32(const float* gy, const float* y, const float* x, const float* wd, const float* s,
                           const float* demod, const uint8_t* label, float* gx, float* gs, int batch, int h, int w,
                           int cin, int cout, int ncls, int up, int act, void* stream);
/* Tensor-core (mma.sync bf16) implementation of e4s_modconv3x3_bwd_f32 for cin % 32 == 0 and cout % 32 == 0.
 * wd_hilo_bf16: [2 (hi, lo)][nphase][9][Cin][Cout] = forward weights with taps flipped, K-major over Cout.
 * When a launch has too few (pixel tile, channel tile) pairs to occupy the GPU, a pair's region passes / parity planes
 * are spread over several CTAs whose partial sums meet in gx by red.global.add: gx is then zeroed first by a memset
 * enqueued on `stream` (no allocation, no synchronisation), and the summation order - hence the last bits of gx -
 * may differ between runs. */
int e4s_modconv3x3_bwd_tc(const float* gy, const float* y, const float* x, const void* wd_hilo_bf16, const float* s,
                          const float* demod, const uint8_t* label, float* gx, float* gs, int batch, int h, int w,
                          int cin, int cout, int ncls, int up, int act, void* stream);
/* Host-only: the work list e4s_modconv3x3_bwd_tc builds for a shape - N-tile width (input channels per work item) and the
 * split of a tile's region passes (gsplit) and parity planes (hsplit) over work items.  ncls: regions of the label map
 * (1 without one).  No launch; testable without a GPU. */
int e4s_modconv3x3_bwd_tc_plan(int batch, int h, int w, int cin, int ncls, int up, int* ntile, int* gsplit, int* hsplit);
/* Host-only: the N-tile width (output channels per work item: 32, 64 or 128) e4s_modconv3x3_tcr_fwd runs a plain (up = 0)
 * layer at.  No launch; testable without a GPU. */
int e4s_modconv3x3_tcr_fwd_plan(int batch, int h, int w, int cout, int* ntile);
/* gdu[b,c,o] += sum over pixels of region c of act'(y)*gy * (act^-1(y) - noise_w*noise - bias): the per-region
 * reduction behind d(loss)/d(demod).  gdu [B, ncls, Cout] is accumulated atomically (caller zeroes it). */
int e4s_class_reduce_f32(const float* gy, const float* y, const uint8_t* label, const float* noise,
                         const float* noise_w, const float* bias, float* gdu, int batch, int ncls, int ho, int wo,
                         int cout, int noise_b, int act, void* stream);
/* Backward of e4s_torgb_fwd_f32 wrt x and s (the skip gradient is an upfirdn2d call).  g: planar [B, 3, H, W]. */
int e4s_torgb_bwd_f32(const float* g, const float* x, const float* wrgb, const float* s, const uint8_t* label,
                      float* gx, float* gs, int batch, int h, int w, int cin, int ncls, void* stream);

/* ---- small fp32 GEMMs: EqualLinear style modulation (model.py:135-169, :276) and LocalMLP (networks.py:15-39) -----------
 * w_is_kn == 0:  y[g, m, n] = act( sum_k x[g, m, k] * w[g, n, k] + bias[g, n] )   (w in nn.Linear layout [N, K]; the caller has
 *                folded EqualLinear's scale / lr_mul into w and bias)
 * w_is_kn != 0:  y[g, m, n] = sum_k x[g, m, k] * w[g, k, n]                        (input gradient of the above; bias must be NULL)
 * act = leaky ReLU with slope act_slope (1 = none).  *_gstride: element strides between groups (0 = shared operand).
 * n % 4 == 0, k % 4 == 0, 16-byte aligned pointers.  workspace: e4s_linear_workspace_floats(groups, m, n, k) floats (may be
 * NULL when that is 0); with a workspace y must be densely packed (y_gstride == m * n). */
int e4s_linear_f32(const float* x, const float* w, const float* bias, float* y, int groups, int m, int n, int k,
                   long long x_gstride, long long w_gstride, long long bias_gstride, long long y_gstride, int w_is_kn,
                   float act_slope, float* workspace, void* stream);
/* Host-only: floats of workspace the two entry points need for a shape (0 = none).  When the output tiles alone cannot fill
 * the GPU, K is cut into slices handled by different CTAs and summed in a fixed order by a second kernel (deterministic). */
long long e4s_linear_workspace_floats(int groups, int m, int n, int k);

/* ---- loss networks of the inversion loop (scripts/optimization.py:88-122) -------------------------------------------
 * Average-pooling pyramid: y2 = 2x2 block means, y4 = 4x4 block means of planar x [planes, H, W] (H % 4 == 0, W % 8 == 0):
 * for a 1024x1024 image these are adaptive_avg_pool2d(x, 512) and (x, 256), the inputs of LPIPS at scales 1 and 2
 * (optimization.py:105-108), of the parsing loss (face_parsing_loss.py:47) and of the identity loss (id_loss.py:26), in
 * one pass over x.  The backward adds the three incoming gradients at full resolution: gx = g1 + up2(g2)/4 + up4(g4)/16
 * (each of g1, g2, g4 may be NULL). */
int e4s_avgpool_pyramid_f32(const float* x, float* y2, float* y4, long long planes, int h, int w, void* stream);
int e4s_avgpool_pyramid_bwd_f32(const float* g1, const float* g2, const float* g4, float* gx, long long planes, int h, int w,
                                void* stream);

/* ---- BiSeNet face parser (src/pretrained/face_parsing/face_parsing_demo.py, model.py, resnet.py) -------------------
 * Bicubic down-sampling of FaceParser.preprocess_img: x planar [B, 3, H, W] -> y planar [B, 3, H/f, W/f], f = factor in
 * {1, 2, 4}, taps [4 f] (BicubicDownSample's normalised kernel), reflect padding of 3 f // 2 rows / columns before and the
 * rest after, the vertical pass first with an fp32 intermediate.  With mean and std ([3] each) the result is then
 * clamp(0, 1) and (v - mean[c]) / std[c]; both NULL: the raw filter output. */
int e4s_bicubic_down_norm_f32(const float* x, const float* taps, const float* mean, const float* std, float* y, int batch,
                              int h, int w, int factor, void* stream);
/* ResNet-18 stem: 7x7 / 2 convolution (3 -> 64, padding 3) + bias + ReLU + 3x3 / 2 max-pool (padding 1).
 * x planar [B, 3, H, W] (H, W multiples of 4); w7x7 [64, 3, 7, 7]; bias [64]; y pixel-major [B, H/4, W/4, 64]. */
int e4s_parser_stem_f32(const float* x, const float* w7x7, const float* bias, float* y, int batch, int h, int w, void* stream);
/* Classifier head: logits = 1x1 convolution (w1x1 [ncls, C], no bias; ncls <= 32, C % 4 == 0) of pixel-major x [B, h, w, C],
 * bilinearly up-sampled (align_corners=True) to out_h x out_w (>= h x w).  logits: planar [B, ncls, out_h, out_w] or NULL;
 * labels: [B, out_h, out_w] first-index argmax over the classes, mapped through lut [256] when lut is given, or NULL. */
int e4s_parse_head_u8(const float* x, const float* w1x1, const uint8_t* lut, uint8_t* labels, float* logits, int batch, int h,
                      int w, int c, int ncls, int out_h, int out_w, void* stream);
/* y[b, c] = mean over the hw pixels of pixel-major x [B, hw, C] (fixed summation order). */
int e4s_channel_mean_f32(const float* x, float* y, int batch, int hw, int c, void* stream);
/* Space-to-depth: x pixel-major [B, H, W, C] -> y [B, H/2, W/2, 4 C], channel (y & 1, x & 1, c) - the operand of a stride-2
 * convolution on the tensor-core kernel (see out_stride 4 of e4s_conv3x3_tcr_f32). */
int e4s_space_to_depth_f32(const float* x, float* y, int batch, int h, int w, int c, void* stream);

/* Layout shuffles between planar and pixel-major (boundary of the module-level API). */
int e4s_planar_to_pixel_f32(const float* x, float* y, int batch, int c, int h, int w, void* stream);
int e4s_pixel_to_planar_f32(const float* x, float* y, int batch, int c, int h, int w, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* E4S_B200_H_ */
