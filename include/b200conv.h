/*
 * b200conv.h -- C ABI of libb200conv.so: the H100 (sm_90a) training hot path behind
 * eladhoffer/convNet.pytorch's trainer.Trainer loop and ResNet-family model factories.
 *
 * The reference has no FFI of its own (it is pure Python on top of torch.nn); every entry point
 * below replaces one implicit torch/cuDNN/ATen operator the reference invokes, cited per function
 * as reference file:line (paths under the reference tree).  INTEGRATION.md shows the ctypes stubs.
 * 54 entry points.
 *
 * Conventions
 *  - every function returns 0 on success or a negative B200_ERR_* code; b200_last_error() gives text.
 *  - all pointers are DEVICE pointers owned by the caller; the library never allocates user tensors.
 *  - activations are NHWC bf16, weights are bf16 [K][R*S][C] ("KRSC"), master weights / gradients /
 *    statistics are fp32.  "stream" is a cudaStream_t; all calls are asynchronous on it.
 *  - there is NO CPU or vendor-library fallback: unsupported shapes return B200_ERR_UNSUPPORTED.
 */
#ifndef B200CONV_H_
#define B200CONV_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* b200_stream_t; /* cudaStream_t */

#define B200_OK 0
#define B200_ERR_INVALID (-1)
#define B200_ERR_UNSUPPORTED (-2)
#define B200_ERR_CUDA (-3)

#define B200_ACT_NONE 0
#define B200_ACT_RELU 1
#define B200_ACT_RELU6 2

/* One convolution problem: x[N,H,W,C] (*) w[K,R,S,C] -> y[N,P,Q,K]; pad_h/pad_w are the LOW pads,
 * P/Q are given explicitly (the high pad is implied).  groups: 1 (dense) or == C == K (depthwise,
 * served by the b200_dwconv_* entry points). */
typedef struct {
  int N, H, W, C;
  int K, R, S;
  int stride;
  int pad_h, pad_w;
  int P, Q;
  /* optional layout of x in ELEMENTS (0 = dense NHWC: C, W*C, H*W*C).  A pixel stride smaller than C makes
   * consecutive "pixels" overlap: the space-to-depth ImageNet stem reads 4 neighbouring 16-channel pixels as
   * one 64-channel pixel this way (only x is affected; y / dy are always dense). */
  int x_pixel_stride, x_row_stride, x_image_stride;
  /* 0: dense.  W > 0 (C == K, C % W == 0, dense x; fprop/dgrad accept W = 64 only, wgrad W = 128 only, any other W is
   * B200_ERR_UNSUPPORTED): block-diagonal convolution -- output channels [W*b, W*b+W) read input channels of the same
   * window only; the weight operand is [K][R*S][W] (fprop), [C][R*S][W] (dgrad), the weight gradient [K][R*S][W].  This
   * is how grouped convolutions with C == K run (b200_group_weight_pack); C != K runs dense on the block-diagonal
   * expansion. */
  int window;
} b200_conv_desc;

typedef struct {
  const float* bias;     /* [K] fp32 or NULL                                   */
  const void* residual;  /* bf16, same shape as the output, added before act; or NULL */
  int act;               /* B200_ACT_*                                         */
  int out_fp32;          /* 1: output is fp32 (logits), 0: bf16                */
  float* bn_stats_workspace; /* non-NULL: also accumulate per-channel sum / sum^2 of the (bf16) output into this BN
                              * workspace (see b200_bn_workspace_floats); finish with b200_bn_finalize.  Needs a
                              * dense bf16 output, K % 64 == 0, no bias/residual/act; else B200_ERR_UNSUPPORTED */
} b200_epilogue;

const char* b200_last_error(void);
int b200_version(void);
/* number of kernels launched by this library in this process (for bench.py's gpu_launches). */
long long b200_launch_count(void);

/* ---- convolution: implicit GEMM on wgmma tensor cores (csrc/conv.cu) ------------------------
 * replaces nn.Conv2d forward            (models/resnet.py:75-78,126-132,226-227; trainer.py:132)
 *          ConvolutionBackward0 (dgrad) (trainer.py:162 loss.backward())
 *          ConvolutionBackward0 (wgrad) (trainer.py:162)
 *          nn.Linear fwd/bwd as a 1x1 conv on a 1x1 map (models/resnet.py:242) */
int b200_conv_fprop(const b200_conv_desc* d, const void* x, const void* w, void* y,
                    const b200_epilogue* ep, b200_stream_t stream);
/* wt is the bf16 weight re-laid as [C][R*S][K]; residual (bf16, shape of dx) may be NULL */
int b200_conv_dgrad(const b200_conv_desc* d, const void* dy, const void* wt, void* dx,
                    const void* residual, b200_stream_t stream);
/* dw fp32 [K][R*S][C]; ACCUMULATES (dw += ...) so that gradient accumulation works.  Split-K over the
 * pixels: partial tiles go to `workspace` (b200_conv_wgrad_workspace_bytes() bytes, any content) and are
 * summed in a fixed order by a second kernel, so the result is deterministic. */
size_t b200_conv_wgrad_workspace_bytes(void);
int b200_conv_wgrad(const b200_conv_desc* d, const void* x, const void* dy, float* dw,
                    void* workspace, size_t workspace_bytes, b200_stream_t stream);

/* ---- depthwise 3x3 convolution, CUDA-core HBM-bound kernels (csrc/dwconv.cu) -------------------
 * replaces nn.Conv2d(groups=C) fwd/bwd (models/mobilenet_v2.py:57-58). w/dw are [R*S][C]. */
int b200_dwconv_fprop(const b200_conv_desc* d, const void* x, const void* w, void* y, b200_stream_t stream);
int b200_dwconv_dgrad(const b200_conv_desc* d, const void* dy, const void* w, void* dx, b200_stream_t stream);
int b200_dwconv_wgrad(const b200_conv_desc* d, const void* x, const void* dy, float* dw,
                      float* workspace, size_t workspace_bytes, b200_stream_t stream);

/* ---- batch norm (csrc/bn.cu) -----------------------------------------------------------------
 * replaces nn.BatchNorm2d train/eval forward + backward (models/resnet.py:88,91,128,130,133,180,228)
 * fused with nn.ReLU / nn.ReLU6 and the residual add (models/resnet.py:115-116,162-163).
 * z: conv output [M][C] bf16.  workspace: fp32, b200_bn_workspace_floats(C) floats. */
size_t b200_bn_workspace_floats(int C);
/* batch statistics -> mean/invstd [C], running stats update (momentum<0: cumulative average with
 * *num_batches_tracked as in Trainer.calibrate_bn, trainer.py:277-285), scale/shift [C] for apply */
int b200_bn_stats(const void* z, long long M, int C, const float* gamma, const float* beta,
                  float eps, float momentum, float* running_mean, float* running_var,
                  long long* num_batches_tracked, float* mean, float* invstd, float* scale, float* shift,
                  float* workspace, b200_stream_t stream);
/* second half of b200_bn_stats for statistics accumulated by b200_conv_fprop (bn_stats_workspace) */
int b200_bn_finalize(long long M, int C, const float* gamma, const float* beta, float eps, float momentum,
                     float* running_mean, float* running_var, long long* num_batches_tracked, float* mean,
                     float* invstd, float* scale, float* shift, float* workspace, b200_stream_t stream);
/* eval mode: scale/shift from running statistics */
int b200_bn_eval_coeffs(int C, const float* gamma, const float* beta, const float* running_mean,
                        const float* running_var, float eps, float* scale, float* shift, b200_stream_t stream);
/* y = act(z*scale+shift + [residual | z2*scale2+shift2]) */
/* act_mask (nullable, b200_bn_act_mask_bytes(M, C) bytes): one bit per element = act'(.) (1 where the activation
 * passes the gradient).  Layout "row quads": the byte of (row, 8-channel vector v8) -- bit c%8 -- is byte row%4 of the
 * 32-bit word (row/4)*(C/8) + v8, so a backward thread fetches the masks of its 2/4/8 consecutive rows with one load.
 * The backward kernels accept it instead of y: 1 bit instead of 16 per element. */
size_t b200_bn_act_mask_bytes(long long M, int C);
int b200_bn_apply(const void* z, long long M, int C, const float* scale, const float* shift,
                  const void* residual, const void* z2, const float* scale2, const float* shift2,
                  int act, void* y, uint8_t* act_mask, b200_stream_t stream);
/* g = dy * act'(a): from act_mask bits when act_mask != NULL, else a = y when y != NULL (a residual was added
 * before the activation), else a is recomputed as z*gamma*invstd + (beta - mean*gamma*invstd) (no read of y).
 * dgamma/dbeta: per-layer sums written to sums[0..C) (dgamma) sums[C..2C) (dbeta) and ACCUMULATED into
 * dgamma_acc/dbeta_acc (gradient arena).  The workspace must be zero before its first use (the kernels
 * leave it zeroed) and must not be shared between concurrently running streams. */
int b200_bn_bwd_reduce(const void* dy, const void* y, const uint8_t* act_mask, const void* z, long long M, int C, int act,
                       const float* mean, const float* invstd, const float* gamma, const float* beta,
                       float* sums, float* dgamma_acc, float* dbeta_acc, float* workspace, b200_stream_t stream);
/* dz = gamma*invstd*(g - dbeta/M - xhat*dgamma/M); optionally also writes g (bf16) for the skip path */
int b200_bn_bwd_dx(const void* dy, const void* y, const uint8_t* act_mask, const void* z, long long M, int C, int act,
                   const float* mean, const float* invstd, const float* gamma, const float* beta,
                   const float* sums, void* dz, void* g_out, b200_stream_t stream);

/* ---- L1 batch norm (csrc/bn_l1.cu) --------------------------------------------------------------
 * replaces L1BatchNorm2d train/eval forward + backward (models/modules/lp_norm.py:238-291, selected by
 * models/resnet.py:393-399 with bn_norm='L1'): per channel mu = mean(z), L = mean|z - mu|,
 * s = 1/(L*sqrt(pi/2) + eps), y = (z - mu)*s*gamma + beta.  b200_bn_apply applies it (scale/shift); the backward
 * is b200_bn_bwd_reduce with invstd = s (dgamma/dbeta sums and arena accumulation) followed by b200_bn_l1_bwd_dx.
 * batch statistics -> mean = mu, invstd = s, sign_sum = sum sign(z - mu) [C], scale/shift [C] for apply; running
 * buffers (nullable) follow the reference: running_mean = running_mean*momentum + mu*(1 - momentum), running_var
 * likewise with s.  Two reads of z, no atomics: the workspace (b200_bn_workspace_floats(C) floats, as for
 * b200_bn_stats) holds per-block partial rows; its accumulators are neither read nor written. */
int b200_bn_l1_stats(const void* z, long long M, int C, const float* gamma, const float* beta, float eps,
                     float momentum, float* running_mean, float* running_var, float* mean, float* invstd,
                     float* sign_sum, float* scale, float* shift, float* workspace, b200_stream_t stream);
/* eval mode: scale = gamma*running_var, shift = beta - running_mean*scale */
int b200_bn_l1_eval_coeffs(int C, const float* gamma, const float* beta, const float* running_mean,
                           const float* running_var, float* scale, float* shift, b200_stream_t stream);
/* dz = gamma*s*(g - sums[C+c]/M) - gamma*s*sqrt(pi/2)*sums[c]/M*(sign(z - mu) - sign_sum/M), sign(0) = 0, with
 * g, y, act_mask, g_out as in b200_bn_bwd_dx and sums from b200_bn_bwd_reduce(..., invstd = s, ...) */
int b200_bn_l1_bwd_dx(const void* dy, const void* y, const uint8_t* act_mask, const void* z, long long M, int C,
                      int act, const float* mean, const float* invstd, const float* sign_sum, const float* gamma,
                      const float* beta, const float* sums, void* dz, void* g_out, b200_stream_t stream);

/* ---- dropout inside residual blocks (csrc/dropout.cu) ---------------------------------------------
 * replaces nn.Dropout(p) after relu(bn1(conv1(x))) of a CIFAR BasicBlock (models/resnet.py:81-118) in training mode.
 * Mask stream: Philox4x32-10 with key {k0, k1} = low / high word of *key (64 bits, device memory: a captured graph reads
 * the value of each replay); the 8-channel vector g = (row*C + c)/8 of dropout layer `layer` uses counter
 * {g & 0xffffffff, g >> 32, layer, 0} and keeps its element j iff ((w[j/2] >> 16*(j%2)) & 0xffff) < T for the four
 * output words w.  T = round((1 - p) * 65536) (T <= 65536), c = fp32(1/(1 - p)).
 * y = keep && pre > 0 ? pre*c : +0 with pre = z*scale + shift; act_mask (required, b200_bn_act_mask_bytes(M, C) bytes,
 * row-quad layout as b200_bn_apply) receives keep && pre > 0. */
int b200_bn_apply_dropout(const void* z, long long M, int C, const float* scale, const float* shift, const uint64_t* key,
                          int layer, unsigned T, float c, void* y, uint8_t* act_mask, b200_stream_t stream);
/* b200_bn_bwd_reduce / b200_bn_bwd_dx of that unit with g = bit ? dy*c : +0 (bits from b200_bn_apply_dropout) */
int b200_bn_bwd_reduce_dropout(const void* dy, const uint8_t* act_mask, const void* z, long long M, int C, float c,
                               const float* mean, const float* invstd, float* sums, float* dgamma_acc, float* dbeta_acc,
                               float* workspace, b200_stream_t stream);
int b200_bn_bwd_dx_dropout(const void* dy, const uint8_t* act_mask, const void* z, long long M, int C, float c,
                           const float* mean, const float* invstd, const float* gamma, const float* sums, void* dz,
                           b200_stream_t stream);

/* ---- pooling (csrc/pool.cu) -------------------------------------------------------------------
 * replaces nn.MaxPool2d(3,2,1) (models/resnet.py:230) and nn.AdaptiveAvgPool2d(1) (resnet.py:241) */
int b200_maxpool3x3s2_fwd(const void* x, int N, int H, int W, int C, void* y, uint8_t* argmax, b200_stream_t stream);
int b200_maxpool3x3s2_bwd(const void* dy, const uint8_t* argmax, int N, int H, int W, int C, void* dx, b200_stream_t stream);
/* ImageNet stem tail bn1 -> relu -> maxpool forward (models/resnet.py:226-230) without materialising the [N,H,W,C]
 * activation: y = maxpool3x3s2(bf16(act(z*scale+shift))) + argmax bytes, bit-identical to b200_bn_apply followed by
 * b200_maxpool3x3s2_fwd. */
int b200_bn_apply_maxpool3x3s2(const void* z, int N, int H, int W, int C, const float* scale, const float* shift,
                               int act, void* y, uint8_t* argmax, b200_stream_t stream);
int b200_avgpool_fwd(const void* x, int N, int HW, int C, void* y, b200_stream_t stream);
int b200_avgpool_bwd(const void* dy, int N, int HW, int C, void* dx, b200_stream_t stream);

/* ---- layout / precision transforms (csrc/prep.cu) ---------------------------------------------
 * replaces inputs.to(device, dtype) (trainer.py:116-117) + the NCHW->NHWC relayout.
 * mode 0: NCHW fp32 -> NHWC bf16 with channels zero-padded to Cpad.
 * mode 1: space-to-depth by 2 for the 7x7/s2 ImageNet stem: out[N,H/2,W/2,Cpad], channel =
 *         (dy*2+dx)*C + c, zero-padded to Cpad (H, W even).
 * mode 2: mode 1 with a physical zero border: out[N, H/2+3, W/2+3, Cpad], data at (+2,+2) -- the 4x4/s1
 *         stem conv (pad 2 low, 1 high) then needs no out-of-bounds handling and can read "wide pixels". */
int b200_input_prep(const float* x_nchw, int N, int C, int H, int W, int Cpad, int mode, void* out, b200_stream_t stream);
/* the same three layouts from uint8 NHWC images [N][H][W][C] (C <= 4), normalised on the fly:
 * value = u8 * scale[c] + bias[c] with scale = 1/(255*std), bias = -mean/std -- ToTensor + Normalize of the reference's
 * preprocess.py:20-24 fused into the relayout (SURVEY.md section 8(f) row 2).  scale_host / bias_host: HOST arrays [C]. */
int b200_input_prep_u8(const uint8_t* x_nhwc, int N, int C, int H, int W, int Cpad, int mode, const float* scale_host,
                       const float* bias_host, void* out, b200_stream_t stream);
/* The same relayouts with the reference Trainer's input mixing (utils/mixup.py:19-26,57-90; trainer.py:119-135) done in
 * the pass.  perm: device int64 [N], the partner sample of each sample.  params: DEVICE parameter block, read by the
 * kernel at run time so that a captured CUDA graph picks up each step's values.  kind:
 *   B200_MIX_NONE   -- exactly b200_input_prep / b200_input_prep_u8 (perm and params may be NULL);
 *   B200_MIX_MIXUP  -- v = lam*x[n] + (1-lam)*x[perm[n]] with two fp32 products and one fp32 sum (no FMA), then one
 *                      rounding to bf16 (bit-exact against the reference's fp32 expression);
 *   B200_MIX_CUTMIX -- pixel (r, c) of sample n is taken from sample perm[n] when r0 <= r < r1 and c0 <= c < c1, else
 *                      from n; in modes 1/2 each of the four sub-pixels of a 2x2 cell decides on its own.
 * uint8 input: each source pixel is normalised (u8*scale+bias, one fmaf) before it is mixed.  The zero border of
 * mode 2 and the channel padding stay zero. */
#define B200_MIX_NONE 0
#define B200_MIX_MIXUP 1
#define B200_MIX_CUTMIX 2
typedef struct {
  float lam;          /* MixUp weight of the sample itself; CutMix: 1 - box area / image area (the loss reads it) */
  int r0, r1, c0, c1; /* CutMix box: rows [r0, r1) x columns [c0, c1) */
} b200_mix_params;
int b200_input_prep_mix(const float* x_nchw, int N, int C, int H, int W, int Cpad, int mode, const long long* perm,
                        const b200_mix_params* params, int kind, void* out, b200_stream_t stream);
int b200_input_prep_u8_mix(const uint8_t* x_nhwc, int N, int C, int H, int W, int Cpad, int mode, const float* scale_host,
                           const float* bias_host, const long long* perm, const b200_mix_params* params, int kind,
                           void* out, b200_stream_t stream);
/* Batch augmentation (the reference's --duplicates with RandomCrop(padding) + RandomHorizontalFlip + ToTensor + Normalize
 * [+ Cutout], preprocess.py:44-54,105-112,159-161,185-227) fused into the mode-0 relayout: uint8 NHWC images
 * x_nhwc [N][H][W][C] (C <= 4) -> out bf16 [N*D][H][W][Cpad].  Output row n' is copy n' % D of image n' / D with the
 * DEVICE draw row params[n'] = int16 {oy, ox, flip, y1, y2, x1, x2, ...} (3 + 4*holes entries per row):
 *   c' = flip ? W-1-c : c,  sy = r + oy - pad,  sx = c' + ox - pad,
 *   u  = (0 <= sy < H && 0 <= sx < W) ? x[n'/D][sy][sx][ch] : 0,   v = lut[ch][u]  (DEVICE fp32 [C][256]),
 *   v  = v * 0.f when y1 <= r < y2 and x1 <= c < x2 for any box, then one rounding to bf16.
 * With lut[ch][u] = ((float)u / 255 - mean[ch]) / std[ch] in fp32 (torchvision's ToTensor + Normalize) the output is
 * b200_input_prep of the reference's augmented fp32 batch, bit for bit.  Any draw values are memory-safe; the kernel
 * reads them at run time, so a captured CUDA graph follows each step's draws. */
int b200_input_prep_u8_aug(const uint8_t* x_nhwc, int N, int D, int C, int H, int W, int Cpad, int pad, const float* lut,
                           const int16_t* params, int holes, void* out, b200_stream_t stream);
/* The same transform with the Resize of the Mix&Match CIFAR size regimes (preprocess.py:44-54 with input_size !=
 * scale_size: RandomCrop(padding) -> Resize -> RandomHorizontalFlip -> ToTensor -> Normalize [-> Cutout]): uint8 NHWC
 * images x_nhwc [N][H][W][C] (C <= 4) -> out bf16 [N*D][OH][OW][Cpad].  Output row n' is copy n' % D of image n' / D
 * with the DEVICE draw row params[n'] = int16 {oy, ox, flip, y1, y2, x1, x2, ...} as above, the boxes in OUTPUT
 * coordinates (Cutout acts on the resized tensor):
 *   w[r][c] = (0 <= r + oy - pad < H && 0 <= c + ox - pad < W) ? x[n'/D][r + oy - pad][c + ox - pad] : 0  (H x W),
 *   p = w resampled to OH x OW exactly as Pillow's 8-bit BILINEAR resize does (the padded zeros are part of the
 *       picture: the filter blends them into the border; horizontal pass into uint8, then the vertical pass),
 *   u = p[r][flip ? OW-1-c : c],   v = lut[ch][u],   v = v * 0.f inside any box, then one rounding to bf16.
 * OH == H && OW == W gives the bytes of b200_input_prep_u8_aug (the filter at scale 1 is the identity).  C <= 4,
 * H, W <= 64, OH, OW <= 128.  Any draw values are memory-safe; the grid depends on N*D only and there is no
 * workspace, so a captured CUDA graph follows each step's images and draws. */
int b200_input_prep_u8_aug_resize(const uint8_t* x_nhwc, int N, int D, int C, int H, int W, int OH, int OW, int Cpad,
                                  int pad, const float* lut, const int16_t* params, int holes, void* out,
                                  b200_stream_t stream);
/* RandomResizedCrop +RandomHorizontalFlip + ToTensor + Normalize of the ImageNet training transform (preprocess.py:71-77,
 * with multi_transform's duplicates, :105-112) fused into the stem relayout.  regions: one DEVICE uint8 buffer of
 * region_bytes bytes holding B uint8 HWC images' regions; index (DEVICE int64 [B][3]) = {byte offset, h, w} of each;
 * draws (DEVICE int32 [B*D][5]) = {y, x, h, w, flip} of each copy's crop box inside its region.  Output row n is copy
 * n % D of image n / D: the crop resampled to OH x OW exactly as Pillow's 8-bit BILINEAR resize does (the crop is the
 * whole image: taps clamp at its edges), mirrored when flip != 0, then v = lut[c][u] (DEVICE fp32 [C][256]) rounded once
 * to bf16.  mode 0: out [B*D][OH][OW][Cpad] (Cpad >= C); mode 2: the padded space-to-depth layout of b200_input_prep
 * (even OH, OW; Cpad >= 4C).  C <= 4, OW <= 512, B*D <= 65535.  Any table values are memory-safe (every read is clamped
 * to its region and to region_bytes); the grid depends on (B*D, OH, OW) only, so a captured graph follows new tables. */
int b200_input_prep_u8_rrc(const uint8_t* regions, long long region_bytes, const long long* index, const int* draws,
                           int B, int D, int C, int OH, int OW, int Cpad, int mode, const float* lut, void* out,
                           b200_stream_t stream);
/* Resize(scale) + CenterCrop(OH x OW) + ToTensor + Normalize of the ImageNet evaluation transform (preprocess.py:20-41,
 * one crop) fused into the stem relayout.  regions: one DEVICE uint8 buffer of region_bytes bytes holding B images'
 * support regions (HWC); index (DEVICE int64 [B][3]) = {byte offset, h, w} of each; geom (DEVICE int32 [B][8]) =
 * {y0, x0, H, W, RH, RW, top, left}: the region's origin in the H x W image, the resized size RH x RW and the crop's
 * origin in the resized image.  Output row n, pixel (o, x) is pixel (top + o, left + x) of image n resized to RH x RW
 * exactly as Pillow's 8-bit BILINEAR resize of the WHOLE image does (image pixel (y, x) is read at (y - y0, x - x0) of
 * the region), or uint8 0 outside the resized image (CenterCrop's padding); then v = lut[c][u] (DEVICE fp32 [C][256])
 * rounded once to bf16.  RH == H, RW == W is the identity (no Resize).  mode 0: out [B][OH][OW][Cpad] (Cpad >= C);
 * mode 2: the padded space-to-depth layout of b200_input_prep (even OH, OW; Cpad >= 4C).  C <= 4, OW <= 512,
 * B <= 65535, any downscale factor.  Any table values are memory-safe (every read is clamped to its region and to
 * region_bytes); the grid depends on (B, OH) only, so a captured graph follows new tables. */
int b200_input_prep_u8_scale_crop(const uint8_t* regions, long long region_bytes, const long long* index,
                                  const int* geom, int B, int C, int OH, int OW, int Cpad, int mode, const float* lut,
                                  void* out, b200_stream_t stream);
/* Baseline JPEG decode into the region buffer of b200_input_prep_u8_rrc / b200_input_prep_u8_scale_crop (csrc/jpeg.cu,
 * tests/jpeg_oracle.py): out receives, for each of the B images, its region (desc words y0, x0, rh, rw) of the RGB
 * image np.asarray(Image.open(f).convert('RGB')) as Pillow (libjpeg-turbo: ISLOW IDCT, fancy upsampling) decodes it,
 * uint8 HWC at byte offset desc[b][26].  payload (DEVICE, 16-byte aligned): the entropy-coded segments, packed Huffman
 * and quantisation tables and the regions the loader decoded on the host, at the offsets of desc (DEVICE int64
 * [B][32], utils/augment.py JpegCollate); intervals (DEVICE int64 [n_intervals][3]) = {image, interval, first byte}
 * of each restart interval.  coef (int16 [coef_blocks][64]) and planes (plane_bytes >= 64 * coef_blocks) are
 * workspaces.  status (DEVICE int32 [B]) is reset, then ORs 1 (bad Huffman code), 2 (premature end of data),
 * 4 (wrong restart marker) or 8 (coefficient index past 63) per image; such an image's pixels are unspecified.  Reads
 * of the entropy-coded data stay inside each image's segment; the descriptor's other offsets are trusted (ops.py
 * jpeg_decode validates them on the host). */
int b200_jpeg_decode(const uint8_t* payload, long long payload_bytes, const long long* desc, int B,
                     const long long* intervals, int n_intervals, int16_t* coef, long long coef_blocks, uint8_t* planes,
                     long long plane_bytes, long long pixels, uint8_t* out, long long out_bytes, int* status,
                     b200_stream_t stream);
/* bf16 [K][T][C] -> bf16 [C][T][K] (dgrad weight layout), multi-tensor: n tensors described by
 * device arrays. */
int b200_weight_transpose(const void* src, void* dst, int K, int T, int C, b200_stream_t stream);
/* all conv weights of a network in one launch: jobs (device) = njobs x {src_off, dst_off, K, T, C, tile_start} ints,
 * offsets in elements from src_base / dst_base, tile_start = running sum of T*ceil(K/32)*ceil(C/32) */
int b200_weight_transpose_batched(const void* src_base, void* dst_base, const int* jobs, int njobs, int total_tiles,
                                  b200_stream_t stream);
/* 7x7/s2/p3 stem weights fp32 [K][7][7][C] -> s2d bf16 [K][4*4][Cpad] and the reverse for wgrad */
int b200_stem_weight_to_s2d(const float* w, int K, int C, int Cpad, void* w_s2d, b200_stream_t stream);
int b200_stem_wgrad_from_s2d(const float* dw_s2d, int K, int C, int Cpad, float* dw, b200_stream_t stream);
int b200_cast_f32_to_bf16(const float* src, void* dst, long long n, b200_stream_t stream);
/* grouped convolution (nn.Conv2d(groups=g), models/resnext.py:10-16): with C == K block diagonal at any window W that is
 * a multiple of the group width and divides C.  pack: fp32 master [K][T][C/g] -> bf16 [K][T][W] (transpose = 0, fprop
 * operand of b200_conv_fprop with desc.window = W) or [C][T][W] (transpose = 1, dgrad operand); unpack: dw_grouped +=
 * the entries of the windowed fp32 gradient [K][T][W] (b200_conv_wgrad with desc.window) that belong to each output
 * channel's group.
 * W == C is the dense block-diagonal expansion, also for C != K (run with desc.window = 0): the fprop operand is
 * [K][T][C], the dgrad operand [C][T][K], and unpack reads a dense [K][T][C] gradient.  Any other W needs C == K. */
int b200_group_weight_pack(const float* w_grouped, int K, int T, int C, int groups, int window, int transpose,
                           void* out_bf16, b200_stream_t stream);
int b200_group_wgrad_unpack(const float* dw_win, int K, int T, int C, int groups, int window, float* dw_grouped,
                            b200_stream_t stream);

/* ---- squeeze-and-excitation on the residual branch (csrc/se.cu) --------------------------------
 * replaces models/modules/se.py:6-25 (SEBlock.forward and its autograd backward) as used by resnet_se / resnext_se
 * (models/resnet.py:112-113,159-160): r' = r * sigmoid(logit[n][c]); the two linear layers in between run on
 * b200_conv_* as 1x1 convolutions on 1x1 maps.  r, g, out: NHWC bf16 [N][HW][C]; logit fp32 [N][C]. */
int b200_se_pool(const void* r, int N, int HW, int C, void* mean_bf16, b200_stream_t stream);
int b200_se_scale_fwd(const void* r, const float* logit, int N, int HW, int C, void* out, b200_stream_t stream);
/* dlogit[n][c] (bf16) = sigma'(logit) * sum_hw g*r  --  gradient of the gate's pre-activation */
int b200_se_bwd_reduce(const void* g, const void* r, const float* logit, int N, int HW, int C, void* dlogit_bf16,
                       b200_stream_t stream);
/* dr = g * sigmoid(logit) + dmean / HW  (dmean bf16 [N][C]: gradient w.r.t. the pooled mean) */
int b200_se_bwd_dx(const void* g, const float* logit, const void* dmean_bf16, int N, int HW, int C, void* dr,
                   b200_stream_t stream);
/* dx = dy * act'(y) for y = act(.), elementwise bf16 (n % 8 == 0) */
int b200_act_bwd(const void* dy, const void* y, long long n, int act, void* dx, b200_stream_t stream);

/* ---- loss (csrc/loss.cu) ----------------------------------------------------------------------
 * replaces utils/cross_entropy.py:14-67 (F.cross_entropy / label smoothing) forward+backward.
 * logits/dlogits rows have pitch ld >= classes (columns [classes, ld) are padding: ignored on read,
 * zeroed in dlogits).  loss != NULL: loss is fp32[3] (device, overwritten): {mean loss, top-1 %, top-5 %} -- the
 * meters of Trainer.forward (trainer.py:224-227, utils/meters.py:59-72: rank of the target class, ties aside) --
 * summed in a fixed order from row_loss (scratch, fp32[2*B]: per-sample loss, per-sample rank of the target).  dlogits != NULL: dlogits (bf16) = grad_scale *
 * (*grad_scale_dev if non-NULL) / B * dloss_i/dlogits -- the device scalar is the upstream gradient of the loss
 * (loss scaling, trainer.py:158-161) so that no host value is baked into a captured graph. */
int b200_softmax_ce(const float* logits, const long long* target, int B, int classes, int ld, float smooth_eps,
                    float grad_scale, const float* grad_scale_dev, float* loss, float* row_loss, void* dlogits_bf16,
                    b200_stream_t stream);
/* soft-target form for MixUp / CutMix (the reference's mix_target + cross_entropy with a float target,
 * utils/mixup.py:37-45, utils/cross_entropy.py:53-54): q = lam*onehot(target[b]) + (1-lam)*onehot(target[perm[b]]),
 * lam = *lam_dev (device: b200_mix_params.lam).  Row loss -(lam*lsm[t] + (1-lam)*lsm[t2]), gradient
 * (lam + (1-lam))*softmax - lam*[c==t] - (1-lam)*[c==t2].  The top-1 / top-5 ranks use target[b] (the meters of the
 * reference read the original target, trainer.py:224).  No smoothing argument: the reference drops label smoothing
 * for soft targets.  Other arguments as b200_softmax_ce. */
int b200_softmax_ce_mix(const float* logits, const long long* target, const long long* perm, const float* lam_dev, int B,
                        int classes, int ld, float grad_scale, const float* grad_scale_dev, float* loss, float* row_loss,
                        void* dlogits_bf16, b200_stream_t stream);
/* column sums of a bf16 [B][K] matrix accumulated into fp32 out[K] (fc bias gradient) */
int b200_colsum_bf16(const void* m, int B, int K, float* out, b200_stream_t stream);

/* ---- optimizer (csrc/optim.cu) ----------------------------------------------------------------
 * replaces Trainer's unscale loop (trainer.py:165-169), WeightDecay.pre_step
 * (utils/regularization.py:127-131), torch.optim.SGD.step (utils/optim.py:254-264) and the
 * fp32->low-precision copy-back (utils/optim.py:43-47,263-264) in ONE pass over flat arenas.
 * Elements [0, wd_count) receive weight decay. hyper: device or host pointer is NOT used; values
 * are passed by value except clip_coef_dev (device scalar multiplied into g, may be NULL).
 * zero_grad != 0: g32 is cleared by a memset behind the update, inside this call (OptimRegime.zero_grad of the NEXT step,
 * utils/optim.py:246-252). */
int b200_fused_sgd(float* p32, float* g32, float* m32, void* p16, long long n, long long wd_count,
                   float lr, float momentum, float dampening, float weight_decay, float inv_scale,
                   const float* clip_coef_dev, int first_step, int zero_grad, b200_stream_t stream);
/* sum of squares of a flat fp32 array -> *out (device, fp32); out is overwritten */
int b200_sumsq(const float* g, long long n, float* out, float* workspace, b200_stream_t stream);
/* GradSmooth (utils/regularization.py:198-224) / clip_grad_norm_ (trainer.py:171-172) on device:
 * mode 0 (clip): coef = min(1, max_norm/(norm+1e-6)); mode 1 (smooth): running = mom*running +
 * (1-mom)*norm (first call: running = norm, coef = 1), coef = running/(norm+1e-6).
 * state[0]=running norm, state[1]=initialised flag; coef_out is a device scalar for fused_sgd. */
int b200_grad_coef(const float* sumsq, float inv_scale, int mode, float max_norm, float momentum,
                   float* state, float* coef_out, float* norm_out, b200_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* B200CONV_H_ */
