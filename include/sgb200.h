/* libsgb200 — C ABI of the H100-native StudioGAN hot path.
 *
 * Everything here is plain C: device pointers, sizes, a cudaStream_t passed as void*.  No torch
 * types cross this boundary.  Every entry point returns 0 on success or an SGB_ERR_* code; nothing
 * throws, nothing allocates behind the caller's back unless the name says "workspace".
 *
 * The reference (POSTECH-CVLab/PyTorch-StudioGAN) has no FFI: its hot path is Python calling
 * torch/cuDNN/cuBLAS ops.  Each entry point below names the reference call site whose arithmetic
 * it replaces (paths relative to the reference checkout, torch/ = installed PyTorch 2.11).
 *
 * Activation layout: NHWC bf16 ("channels-last"); element (b,h,w,c) of a tensor with channel
 * stride cs lives at base + ((b*H + h)*W + w)*cs + c.  Master weights / statistics / sigma: fp32.
 */
#ifndef SGB200_H_
#define SGB200_H_
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SGB_OK 0
#define SGB_ERR_ARG 1
#define SGB_ERR_CUDA 2
#define SGB_ERR_UNSUPPORTED 3

typedef void* sgb_stream_t; /* cudaStream_t */

/* library / device probe: returns the ABI version (or -1), no GPU work. */
int sgb_abi_version(void);
/* 0 if a sm_90 device is current and usable, SGB_ERR_UNSUPPORTED on another architecture, else SGB_ERR_CUDA. */
int sgb_device_check(void);
/* Make ``device``'s primary context current on the calling host thread (call once per thread that uses the library,
 * e.g. PyTorch autograd worker threads). */
int sgb_bind_device(int32_t device);

/* ------------------------------------------------------------------------------------------
 * Implicit-GEMM convolution on Hopper tensor cores (TMA-staged NHWC tiles, wgmma, register accumulators).
 * Stride-1 convolution with KHxKW taps and zero padding; H,W are the OUTPUT spatial size
 * (== input size).  Also serves linear layers (H=W=1) and dgrad (caller passes the
 * transposed/flipped packed weights).
 * Replaces: nn.Conv2d / nn.Linear forward and input-gradient as used by
 *   src/utils/ops.py:165-173,187-188,195-204,219-220 and every conv2d / linear call in
 *   src/models/big_resnet_deep_legacy.py:49-73,210-229, src/models/big_resnet.py, src/models/resnet.py.
 * ------------------------------------------------------------------------------------------ */
typedef struct sgb_conv_desc {
  int32_t B, H, W;
  int32_t Cin, Cout;
  int32_t KH, KW, pad_h, pad_w;
  const void* x;       /* bf16 NHWC input */
  int64_t x_cstride;   /* elements between consecutive pixels (>= Cin, multiple of 8) */
  const void* w;       /* bf16 packed weights [Cout][KH*KW][Cin] (w_mode 0) */
  int32_t w_mode;      /* 0: shared weights; 1: per-image B operand [B][Cout][Cin]; 2: per-image, Cout-contiguous
                          [B][Cin][Cout] (MN-major).  Modes 1/2 (batched GEMM for attention) need KH=KW=1, H*W >= 128 */
  float alpha;         /* accumulator scale */
  const float* alpha_ptr; /* optional device scalar multiplied into alpha */
  const float* bias;   /* fp32 [Cout] or NULL */
  const void* residual;/* bf16 NHWC or NULL; added after bias */
  int64_t res_cstride;
  int32_t res_up2;     /* 1: residual is at half resolution, read at (h/2, w/2) (nearest x2 upsample) */
  int32_t res_after_mask; /* 0: residual added before relu/mask; 1: added last (skip-branch gradient in dgrad) */
  const void* mask;    /* bf16 NHWC or NULL; output is zeroed where mask <= 0 (ReLU backward) */
  int64_t mask_cstride;
  int32_t relu;        /* 1: ReLU applied last (before mask) */
  void* y;             /* output, bf16 (or fp32 if y_fp32) */
  int64_t y_cstride;
  int32_t y_fp32;
  /* Generalisations used by the InceptionV3 feature extractor (src/metrics/inception_net.py); 0 = plain same-size conv.
   * Hin/Win: input spatial size when it differs from the output grid H x W ("valid" convolutions: H = Hin - KH + 1 + 2 pad).
   * out_sub = 2: only the even (h, w) positions of the H x W grid are stored, at (h/2, w/2) of a ceil(H/2) x ceil(W/2)
   * tensor, i.e. a stride-2 convolution computed on the stride-1 grid (four layers of the network). */
  int32_t Hin, Win;
  int32_t out_sub;
  float res_scale;     /* residual multiplier (0 is read as 1): 0.25 with res_up2 = the backward of a 2x2 average pooling
                          added in the epilogue (src/models/big_resnet_deep_legacy.py:220-224, the pooled skip branch) */
  /* ReLU masks as bit planes (Cout % 64 == 0, bf16 output): [B*H*W][Cout/64] 64-bit words, bit j of word c = channel 64c + j.
   * relu_bits (needs relu = 1): written next to y, bit = (y > 0);  mask_bits: used instead of ``mask`` (1/16 of its bytes) by
   * the input-gradient launch of the layer that consumed y (the in-place d_act_fn of src/config.py:486 in backward). */
  const void* mask_bits;
  void* relu_bits;
  /* Row softmax of the attention map (src/utils/ops.py:93-97) inside the GEMM epilogue, 1x1 / w_mode 1 launches with
   * Cout = keys (multiple of 64), bf16 output, no other epilogue operand:
   *   sm_mode 1: statistics pass -- nothing is stored to y; sm_stats[row][part] = (max, sum exp(. - max)) over the columns of one
   *              output-channel tile (128 channels; 64 when Cout = 64); parts per row = sgb_conv_softmax_parts(desc)
   *   sm_mode 2: y = exp(acc - m_row) / l_row with (m, l) merged from sm_stats (the same GEMM launched a second time)
   *   sm_mode 3: y = sm_p * (acc - sm_delta[row]): softmax backward dS = P * (dP - delta), delta = rowsum(dO * O) */
  int32_t sm_mode;
  float* sm_stats;
  const float* sm_delta;
  const void* sm_p;     /* bf16 NHWC, same shape as y */
  int64_t sm_p_cstride;
} sgb_conv_desc;

int sgb_conv_fprop(const sgb_conv_desc* d, sgb_stream_t stream);

/* Weight gradient: dw[co][tap][ci] += sum_{b,h,w} dy[b,h,w,co] * x[b,h+kh-pad,w+kw-pad,ci]
 * (wgmma with MN-major operands, split over pixels, fp32 atomics into dw).
 * Replaces: conv/linear weight-gradient of torch autograd for the same call sites. */
typedef struct sgb_wgrad_desc {
  int32_t B, H, W;
  int32_t Cin, Cout;
  int32_t KH, KW, pad_h, pad_w;
  const void* x;
  int64_t x_cstride;
  const void* dy;
  int64_t dy_cstride;
  float* dw;          /* fp32 [Cout][KH*KW][Cin]  (per_image: [B][Cout][KH*KW][Cin]) */
  int32_t accumulate; /* 0: dw is zeroed first */
  int32_t per_image;  /* 1: one gradient per image (attention dK/dV); needs H*W >= 128 */
  float* dbias;       /* optional fp32 [Cout]: bias gradient sum_{b,h,w} dy, produced by the same launch (zeroed first unless
                         accumulate): a constant-ones operand rides along the dy tiles on the tensor pipe, so no separate
                         reduction pass reads dy -- only when sgb_conv_wgrad_fuses_dbias(d) returns 1 (not per_image) */
} sgb_wgrad_desc;

int sgb_conv_wgrad(const sgb_wgrad_desc* d, sgb_stream_t stream);
/* 1 if sgb_conv_wgrad(d) can also deliver d->dbias (3x3 / 64-channel kernel: constant-one operand atom in the otherwise
 * idle half of its last MMA group; generic kernel: an N = 16 ones-product on its first-tap / first-channel-tile work
 * items); 0 for per-image gradients. */
int sgb_conv_wgrad_fuses_dbias(const sgb_wgrad_desc* d);

/* ------------------------------------------------------------------------------------------
 * Spectral normalisation (power iteration + sigma) and tensor-core weight packs.
 * Replaces: torch.nn.utils.spectral_norm forward-pre-hook (torch/nn/utils/spectral_norm.py:62-114)
 *   installed by src/utils/ops.py:195-224 (eps = 1e-6, one iteration, dim = 0).
 * W is the module weight viewed as [R = out_channels][K = in_channels*kh*kw], fp32.
 * ws: caller-owned fp32 workspace of sgb_sn_workspace_floats(R, K) floats, ZERO-initialised once.
 * ------------------------------------------------------------------------------------------ */
int64_t sgb_sn_workspace_floats(int32_t R, int32_t K);
/* do_power_iteration=1: v <- normalize(W^T u), u <- normalize(W v) in place; always: *sigma = u.(W v). */
int sgb_sn_power_iter(const float* W, float* u, float* v, float* sigma, float* ws, int32_t R, int32_t K, float eps,
                      int32_t do_power_iteration, sgb_stream_t stream);
/* Packs W[Cout][Cin][taps] / sigma (sigma may be NULL = 1) into bf16:
 *   w_fprop[Cout][taps][Cin] and/or w_dgrad[Cin][taps (rotated 180 deg)][Cout].
 * perm_S > 1: output rows re-ordered (row c*S+s -> s*C+c) so that linear0's result is NHWC
 *   (src/models/big_resnet_deep_legacy.py:167-168 views it as [C, 4, 4]). */
/* Cout_p / Cin_p >= Cout / Cin are the (zero-padded, caller-zeroed) pack extents, e.g. 3 -> 8 for image convs. */
int sgb_weight_pack(const float* W, const float* sigma, void* w_fprop, void* w_dgrad, int32_t Cout, int32_t Cin,
                    int32_t taps, int32_t perm_S, int32_t Cout_p, int32_t Cin_p, sgb_stream_t stream);
/* Batched form: all layers of a network in three launches.  ``table`` is a DEVICE array of sgb_sn_layer; per layer it
 * runs the power iteration (has_sn) and writes sigma_all[layer] (1 for layers without spectral norm), then emits the packs
 * at pack_f + off_f / pack_d + off_d (element offsets, bf16; caller zero-fills padded extents; pack_d may be NULL).
 * max_blocks_*: grid.x of the three kernels (>= the largest per-layer need, see sgb200/snbatch.py). */
typedef struct sgb_sn_layer {
  const float* W;
  float* u;
  float* v;
  float* ws;
  int32_t R, K;
  int32_t Cout, Cin, taps, perm_S, Cout_p, Cin_p;
  int64_t off_f, off_d;
  int32_t has_sn;
  int32_t tile_start;  /* pack work units (~1024 weights) of the layers before this one: taps*ceil(Cout/32)*ceil(Cin/32) per
                          layer (taps <= 9), else 4*ceil(Cout*Cin*taps/4096) */
} sgb_sn_layer;
/* Partials per row the softmax statistics pass of sgb_conv_fprop writes for this problem size (2 x channel tiles). */
int sgb_conv_softmax_parts(const sgb_conv_desc* d);
/* Discriminator head on the fp32 sum-pooled features h [B][C] (src/models/big_resnet_deep_legacy.py:346-349,366-368; identical
 * in big_resnet.py / resnet.py): adv[b] = <h_b, w1> / sigma1 + b1 + <h_b, E[labels[b]]> / sigmaE.  sigma1 / sigmaE / b1: device
 * scalars or NULL; E NULL: unconditional head.  Backward: dh [B][C]; gw1 [C] and gE [n_cls][C] are the gradients of the
 * EFFECTIVE (spectrally normalised) weights -- gE is ADDED to (zero it first), gw1 / db1 are overwritten -- and go through
 * sgb_sn_backward like every other layer's. */
int sgb_dhead_fwd(const float* h, const float* w1, const float* sigma1, const float* b1, const float* E, const float* sigmaE,
                  const int64_t* labels, int32_t B, int32_t C, float* adv, sgb_stream_t stream);
int sgb_dhead_bwd(const float* dadv, const float* h, const float* w1, const float* sigma1, const float* E, const float* sigmaE,
                  const int64_t* labels, int32_t B, int32_t C, float* dh, float* gw1, float* gE, float* db1, sgb_stream_t stream);
/* out[r] = sum_c x[r][c] * y[r][c] (bf16 rows of C channels, fp32 out): delta of the softmax backward. */
int sgb_rowdot(const void* x, int64_t xs, const void* y, int64_t ys, int64_t rows, int32_t C, float* out, sgb_stream_t stream);
/* max_blocks_wtu / max_blocks_wv: grid width of the two power-iteration launches; total_pack_tiles: sum of the table's pack
 * work units (the pack launch walks one global unit index, see tile_start). */
int sgb_sn_batch(const sgb_sn_layer* table, int32_t n_layers, float* sigma_all, void* pack_f, void* pack_d, float eps,
                 int32_t do_power_iteration, int32_t max_blocks_wtu, int32_t max_blocks_wv, int32_t total_pack_tiles,
                 sgb_stream_t stream);
/* dW[Cout][Cin][taps] (=|+=) (G - <G, W/sigma> u v^T) / sigma with G in the fprop-pack layout (fp32, from
 * sgb_conv_wgrad).  sigma NULL: plain re-layout of G (layers without spectral norm). */
int sgb_sn_backward(const float* G, const float* W, const float* u, const float* v, const float* sigma,
                    float* scratch_dot, float* dW, int32_t Cout, int32_t Cin, int32_t taps, int32_t perm_S,
                    int32_t Cin_p, int32_t accumulate, sgb_stream_t stream);

/* Batched form of sgb_sn_backward: every layer of one network pass in two launches.  ``table`` is a DEVICE array;
 * layer l reads its weight gradient at g_flat + off_g (fprop-pack layout, fp32), the u / v / sigma copies of that forward
 * pass at u_flat + off_u, v_flat + off_v, sigma_all[l], and ADDS to dW (NULL: layer skipped).  dots: fp32 [n_layers]
 * scratch (zeroed here). */
typedef struct sgb_snbwd_layer {
  const float* W;
  float* dW;
  int64_t off_g, off_u, off_v;
  int32_t Cout, Cin, taps, perm_S, Cin_p, has_sn;
} sgb_snbwd_layer;
int sgb_sn_backward_batch(const sgb_snbwd_layer* table, int32_t n_layers, const float* g_flat, const float* sigma_all,
                          const float* u_flat, const float* v_flat, float* dots, int32_t max_blocks, sgb_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Batch-norm family (NHWC bf16 activations, fp32 statistics).
 * Replaces: ops.ConditionalBatchNorm2d.forward (src/utils/ops.py:24-28), ops.batchnorm_2d (:227-228),
 *   F.batch_norm fwd/bwd; the [sum, sumsq, count] / [S1, S2] vectors are the cross-rank reduction points of
 *   torch.nn.SyncBatchNorm (torch/nn/modules/_functions.py:7-212) and src/sync_batchnorm/batchnorm.py:94-175.
 * ------------------------------------------------------------------------------------------ */
int sgb_bn_stats(const void* x, int64_t npix, int32_t C, int64_t x_cstride, float* sum, float* sumsq, sgb_stream_t stream);
/* mode 0: cBN (gain/bias [nb=B][C], scale = rstd*(1+gain)); 1: affine (gain=weight[C], bias[C], nb=1); 2: plain (nb=1). */
int sgb_bn_finalize(const float* sum, const float* sumsq, float count, float* running_mean, float* running_var,
                    float momentum, float eps, int32_t use_batch_stats, int32_t track, int32_t mode, const float* gain,
                    const float* bias, int32_t nb, int32_t C, float* mean, float* rstd, float* scale, float* shift,
                    int64_t affine_ld, sgb_stream_t stream);   /* affine_ld: floats between the rows of the per-image gain / bias
                                                                  (0 = C; > C when they are column slices of one batched GEMM output) */
/* y = [relu](x*scale + shift); per_image: scale/shift are [B][C] else [C]; up2: y is the nearest x2 upsample. */
int sgb_scale_shift_act(const void* x, int32_t B, int32_t H, int32_t W, int32_t C, int64_t x_cstride, const float* scale,
                        const float* shift, int32_t per_image, int32_t relu, int32_t up2, void* y, int64_t y_cstride,
                        sgb_stream_t stream);
/* s1[b,c] = sum dz, s2[b,c] = sum dz*xhat, S1[c] = sum_b g1*s1, S2[c] = sum_b g1*s2 (g1 = scale/rstd). */
int sgb_bn_bwd_reduce(const void* dy, int64_t dy_cstride, const void* x, int64_t x_cstride, int32_t B, int32_t H, int32_t W,
                      int32_t C, const float* scale, const float* shift, int32_t per_image, const float* mean,
                      const float* rstd, int32_t relu, int32_t up2, float* s1, float* s2, float* S1, float* S2,
                      sgb_stream_t stream);
int sgb_bn_bwd_apply(const void* dy, int64_t dy_cstride, const void* x, int64_t x_cstride, int32_t B, int32_t H, int32_t W,
                     int32_t C, const float* scale, const float* shift, int32_t per_image, const float* mean,
                     const float* rstd, const float* S1, const float* S2, float count, int32_t relu, int32_t up2,
                     int32_t use_batch_stats, void* dx, int64_t dx_cstride, sgb_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Element-wise / small reductions (NHWC bf16 unless noted).  Reference call sites: ReLU, AvgPool2d(2),
 * F.interpolate(nearest), residual adds in src/models/big_resnet_deep_legacy.py:49-73,210-229,334-345;
 * MaxPool2d / Softmax / sigma*attn_g in src/utils/ops.py:79-103; nn.Tanh at big_resnet_deep_legacy.py:183.
 * ------------------------------------------------------------------------------------------ */
/* out = act(a*[*a_dev]*x + b*y), then masked by (mask > 0) if mask; act 0 none / 1 relu. */
int sgb_axpby(const void* x, int64_t xs, const void* y, int64_t ys, const void* mask, int64_t ms, void* out, int64_t os,
              int64_t npix, int32_t C, float a, const float* a_dev, float b, int32_t act, sgb_stream_t stream);
/* 2x2 pooling to [B,Ho,Wo,C]; mode 0 average, 1 max, 2 sum (the gradient of a nearest x2 up-sampled residual). */
int sgb_pool2_fwd(const void* x, int64_t xs, void* y, int64_t ys, int32_t B, int32_t Ho, int32_t Wo, int32_t C, int32_t mode,
                  sgb_stream_t stream);
/* dx = pool2 backward of dy (+ add) (masked by relu_src > 0); x needed for max (first max in scan order wins).
 * rs == -1: relu_src holds the bit planes a relu conv epilogue wrote (sgb_conv_desc.relu_bits) instead of the bf16 tensor. */
/* a0 = relu(x) (full resolution) and y = 2x2 average of a0, one pass: entry of a down-sampling discriminator block
 * (self.activation + self.average_pooling on the skip, src/models/big_resnet_deep_legacy.py:211-224,
 * src/models/big_resnet_deep_studiogan.py:233-249). */
int sgb_relu_pool2(const void* x, int64_t x_cstride, void* a0, int64_t a0_cstride, void* y, int64_t y_cstride, int32_t B,
                   int32_t Ho, int32_t Wo, int32_t C, sgb_stream_t stream);
int sgb_pool2_bwd(const void* dy, int64_t dys, const void* x, int64_t xs, const void* add, int64_t adds, const void* relu_src,
                  int64_t rs, void* dx, int64_t dxs, int32_t B, int32_t Ho, int32_t Wo, int32_t C, int32_t mode,
                  sgb_stream_t stream);
int sgb_softmax_rows(const void* s, void* p, int64_t rows, int32_t n, sgb_stream_t stream);
int sgb_softmax_bwd_rows(const void* p, const void* dp, void* ds, int64_t rows, int32_t n, sgb_stream_t stream);
int sgb_dot(const void* x, const void* y, int64_t n, float* out, sgb_stream_t stream);
/* h[b,c] = sum_hw act(x) (fp32): discriminator head sum-pool (big_resnet_deep_legacy.py:344-345). */
int sgb_sum_hw(const void* x, int64_t xs, int32_t B, int32_t HW, int32_t C, int32_t relu, float* h, sgb_stream_t stream);
int sgb_sum_hw_bwd(const float* dh, const void* x, int64_t xs, void* dx, int64_t dxs, int32_t B, int32_t HW, int32_t C,
                   int32_t relu, sgb_stream_t stream);
/* image layout converters: NCHW fp32 <-> NHWC bf16 (channels zero-padded to Cp); act 1 = tanh. */
int sgb_img_to_nhwc(const float* img, void* out, int32_t B, int32_t C, int32_t HW, int32_t Cp, sgb_stream_t stream);
int sgb_nhwc_to_img(const void* in, int32_t in_fp32, int64_t cs, float* img, int32_t B, int32_t C, int32_t HW, int32_t act,
                    sgb_stream_t stream);
int sgb_img_grad_to_nhwc(const float* dimg, const float* y, void* out, int32_t B, int32_t C, int32_t HW, int32_t Cp,
                         sgb_stream_t stream);
/* 3x3 / pad-1 patch gather of a 3-channel image into [B,H,W,32] bf16 (k = tap*3 + c, 27..31 zero) and its adjoint:
 * the 3 -> C input convolution (input_conv, src/models/big_resnet_deep_legacy.py:259) becomes a K = 32 GEMM. */
int sgb_col27(const void* src, int32_t src_nchw_f32, int64_t cs, void* out, int32_t B, int32_t H, int32_t W, sgb_stream_t stream);
int sgb_col27_bwd(const void* dcol, float* dimg, int32_t B, int32_t H, int32_t W, sgb_stream_t stream);
/* Inception pooling: 3x3, stride 1|2, pad 0|1; mode 0 = average with count_include_pad=False, 1 = max
 * (src/metrics/inception_net.py:86,91,153,178,208,241). */
int sgb_pool3x3(const void* x, int64_t xs, void* y, int64_t ys, int32_t B, int32_t H, int32_t W, int32_t C, int32_t stride,
                int32_t pad, int32_t mode, sgb_stream_t stream);
/* out[B][2H][2W][C]: out[b,2h,2w,:] = x[b,h,w,:], zero elsewhere (NHWC bf16): the adjoint of a stride-2 sub-sampling.  With
 * it DCGAN's ConvTranspose2d / Conv2d (kernel 4, stride 2, padding 1; src/models/deep_conv.py:20,140) run on the stride-1
 * conv engine: conv_transpose(x) = conv_same_4x4(zero_stuff(x)), and the strided conv's gradients see zero_stuff(dy). */
int sgb_zero_stuff2(const void* x, int64_t xs, void* y, int64_t ys, int32_t B, int32_t H, int32_t W, int32_t C, sgb_stream_t stream);
/* uint8 quantisation of generated images, bit-exact with ops.quantize_images (src/utils/ops.py:251-255). */
int sgb_quantize_u8(const float* img, uint8_t* out, int64_t n, sgb_stream_t stream);
/* Fused evaluation pre-processing on the device (quantise -> bilinear resize to SxS -> /255 -> (x-0.5)/0.5;
 * src/utils/ops.py:251-263, src/utils/resize.py:50-94, src/metrics/preparation.py:103-122).  img: NCHW fp32 [B,3,H,W].
 * resizer 0 = "legacy" (torch F.interpolate bilinear, align_corners=False, clipped to [0,255]; resize.py:83-91),
 *         1 = "friendly" (PIL bilinear on float32 'F'-mode channels, anti-aliased when shrinking; resize.py:50-53,72-82).
 * out_img (optional): NCHW fp32 [B,3,S,S]; out_col (optional): [B,So,So,32] bf16 stride-2 valid 3x3 patches, So=(S-3)/2+1. */
int sgb_quantize_resize_normalize(const float* img, int32_t quantize, int32_t B, int32_t H, int32_t W, int32_t S, float* out_img,
                                  void* out_col, int32_t resizer, sgb_stream_t stream);
/* Data path: uint8 NHWC [B,H,W,3] (HDF5 "imgs" / decoded folders, src/data_util.py:59-142, src/utils/hdf5.py) -> NCHW fp32 in
 * [-1,1], i.e. RandomHorizontalFlip (flip[b] != 0; flip may be NULL) + ToTensor + Normalize(0.5, 0.5) of the reference's
 * per-sample transform chain, bit-identical, on the device. */
int sgb_u8_to_img(const uint8_t* u8, const uint8_t* flip, float* img, int32_t B, int32_t H, int32_t W, sgb_stream_t stream);
int sgb_cast_f32_to_bf16(const float* in, void* out, int64_t n, float scale, sgb_stream_t stream);
int sgb_cast_bf16_to_f32(const void* in, float* out, int64_t n, sgb_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Optimiser: fused Adam (torch.optim.Adam, eps 1e-6 at src/config.py:541-563) + EMA lerp
 * (src/utils/ema.py:27-40) over a flat fp32 parameter arena.  ema may be NULL.
 * ------------------------------------------------------------------------------------------ */
int sgb_adam_ema_step(float* p, const float* g, float* m, float* v, int64_t n, float lr, float beta1, float beta2, float eps,
                      int32_t step, const int32_t* step_dev, float* ema, float ema_decay, float grad_scale, sgb_stream_t stream);
/* step_dev (optional): int32 step counter in device memory used for the bias corrections instead of `step`, so that a
 * captured CUDA graph of the update stays correct when replayed. */
int sgb_ema_lerp(float* ema, const float* p, int64_t n, float decay, sgb_stream_t stream);
/* WGAN weight clipping (replaces src/worker.py:490-492, p.data.clamp_(-c, c) per discriminator parameter): x clamped to
 * [-c, c] in place over a flat fp32 arena, NaN propagated as torch.clamp does; c >= 0 (the arena's zero padding stays 0). */
int sgb_clamp(float* x, int64_t n, float c, sgb_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Gradient penalty (replaces utils/losses.py:268-275 cal_deriv + :301-316 cal_grad_penalty).
 * The second-order term is evaluated as "reverse over forward": P = mean_b (||g_b|| - 1)^2 with g = d(sum adv)/dx_hat;
 * dP/dtheta = d/dtheta <v, g(theta)> for the constant seed v = dP/dg, and <v, g> is the directional derivative of the
 * discriminator along v, i.e. the output of a tangent (JVP) pass.  Kernels: interpolation, per-sample norms, the seed,
 * and the (x, tangent, gamma) derivatives of a training-mode batch norm's tangent map (torch's
 * batchnorm_double_backward).  All other layers' tangent maps are the forward kernels above (convolutions are linear).
 *   sums layout: [5][C] = sum a, sum c, sum xhat*a, sum xhat*c, sum a*c   (a = tangent, c = incoming cotangent)
 * ------------------------------------------------------------------------------------------ */
int sgb_gp_interpolate(const float* real, const float* fake, const float* alpha, float* out, int32_t B, int64_t n_per,
                       sgb_stream_t stream);
int sgb_gp_sumsq(const float* g, float* sumsq, int32_t B, int64_t n_per, sgb_stream_t stream);
int sgb_gp_seed(const float* g, const float* sumsq, float* v, int32_t B, int64_t n_per, sgb_stream_t stream);
/* Max-gradient penalty (replaces utils/losses.py:337-353 cal_maxgrad_penalty): *penalty = P = max_b sumsq[b] and the seed
 * v = dP/dg = 2 g_b / n_ties on the samples whose sumsq equals the maximum, 0 elsewhere (torch's backward of a full max()
 * reduction splits the gradient evenly over ties).  sumsq: the per-sample output of sgb_gp_sumsq. */
int sgb_gp_seed_max(const float* g, const float* sumsq, float* v, float* penalty, int32_t B, int64_t n_per, sgb_stream_t stream);
/* DRAGAN perturbation (replaces utils/losses.py:319-335 cal_dra_penalty up to the discriminator call):
 * sgb_dra_std: *sigma = real_images.std() (unbiased, over all n elements; fp64 accumulation, one fp32 result on the
 *   device).  ws: fp64 scratch of 2 * SGB_DRA_STD_PARTS elements.
 * sgb_dra_perturb: out = real + alpha[b] * ((0.5 * *sigma) * noise), rounded as torch evaluates that expression; alpha [B]
 *   and noise (shaped like real) are the reference's host draws. */
#define SGB_DRA_STD_PARTS 256
int sgb_dra_std(const float* x, int64_t n, double* ws, float* sigma, sgb_stream_t stream);
int sgb_dra_perturb(const float* real, const float* sigma, const float* alpha, const float* noise, float* out, int32_t B,
                    int64_t n_per, sgb_stream_t stream);
int sgb_bn_tangent_bwd_reduce(const void* x, int64_t x_cstride, const void* a, int64_t a_cstride, const void* c, int64_t c_cstride,
                              int64_t npix, int32_t C, const float* mean, const float* rstd, float* sums, sgb_stream_t stream);
int sgb_bn_tangent_bwd_apply(const void* x, int64_t x_cstride, const void* a, int64_t a_cstride, const void* c, int64_t c_cstride,
                             int64_t npix, int32_t C, const float* gamma, const float* mean, const float* rstd,
                             const float* sums, float count, int32_t use_batch_stats, void* dx, int64_t dx_cstride, void* da,
                             int64_t da_cstride, sgb_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Augmentations on NCHW fp32 images (csrc/augment.cu).
 * Replaces: diffaug.apply_diffaug, policy "color,translation,cutout" (src/utils/diffaug.py:37-100) -- seven tensor-op passes in
 *   the reference, one gather kernel here -- and cr.apply_cr_aug (src/utils/cr.py:13-50).
 * params: fp32 [B][7] = {brightness offset, saturation factor, contrast factor, shift_h, shift_w, cutout_h0, cutout_w0}.
 * ------------------------------------------------------------------------------------------ */
int sgb_sample_mean(const float* x, int32_t B, int64_t n_per, float* out, sgb_stream_t stream);
int sgb_diffaug_fwd(const float* x, const float* params, const float* mean_x, float* y, int32_t B, int32_t H, int32_t W,
                    int32_t do_color, int32_t do_translation, int32_t do_cutout, sgb_stream_t stream);
/* adjoint of sgb_diffaug_fwd; mean_ws: fp32 [B] scratch. */
int sgb_diffaug_bwd(const float* dy, const float* params, float* dx, float* mean_ws, int32_t B, int32_t H, int32_t W,
                    int32_t do_color, int32_t do_translation, int32_t do_cutout, sgb_stream_t stream);
/* y[b,c,h,w] = xf[b,c,reflect(h + tx[b]),reflect(w + ty[b])], xf = x mirrored along w where flip[b] (any of the three may be NULL). */
int sgb_cr_aug(const float* x, const uint8_t* flip, const int32_t* tx, const int32_t* ty, float* y, int32_t B, int32_t C, int32_t H,
               int32_t W, sgb_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Evaluation metrics in fp64 on the device (csrc/metrics.cu).
 * Replaces: fid.calculate_moments / np.mean + np.cov (src/metrics/fid.py:65-98) and prdc.compute_prdc's three
 *   sklearn pairwise_distances matrices + argpartition (src/metrics/prdc.py:87-168).
 * ------------------------------------------------------------------------------------------ */
/* sum[D] += sum_r f[r], outer[D][D] (upper-triangular 64x64 blocks only) += sum_r f[r] f[r]^T for a batch of n fp32
 * feature rows; sum / outer are caller-zeroed fp64 accumulators (the cross-rank reduction point of SURVEY 8e). */
int sgb_feat_moments_accumulate(const float* feats, int32_t n, int32_t D, double* sum, double* outer, sgb_stream_t stream);
/* mu = sum / n, sigma = (outer - n mu mu^T) / (n - 1) as a full symmetric matrix (np.cov(rowvar=False)). */
int sgb_feat_moments_finalize(const double* sum, const double* outer, double n, int32_t D, double* mu, double* sigma,
                              sgb_stream_t stream);
/* radii[i] = distance from x_i to its nearest_k-th neighbour among the rows of x (self counted as the 0-th):
 * prdc.compute_nearest_neighbour_distances (src/metrics/prdc.py:115-126).  x: fp64 [n][D]; sqnorm_ws: fp64 [n], receives
 * the squared row norms (re-used by sgb_prdc_cross); nearest_k <= 7. */
int sgb_prdc_radii(const double* x, int32_t n, int32_t D, int32_t nearest_k, double* sqnorm_ws, double* radii,
                   sgb_stream_t stream);
/* Real-to-fake distance tiles reduced on the fly (src/metrics/prdc.py:129-168):
 *   col_count[j] = #{i : d(real_i, fake_j) < radii_real[i]}   -> precision = mean(col_count > 0), density = mean(col_count) / k
 *   row_any[i]   = any_j d(real_i, fake_j) < radii_fake[j]    -> recall
 *   row_cov[i]   = min_j d(real_i, fake_j) < radii_real[i]    -> coverage */
int sgb_prdc_cross(const double* real, const double* real_sqnorm, const double* fake, const double* fake_sqnorm,
                   const double* radii_real, const double* radii_fake, int32_t n_real, int32_t n_fake, int32_t D,
                   int32_t* col_count, uint8_t* row_any, uint8_t* row_cov, sgb_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* SGB200_H_ */
