/*
 * bbb_b200.h -- C ABI of the H100-native Bayes-by-Backprop layer engine.
 *
 * The reference (kumar-shridhar/PyTorch-BayesianCNN) has no FFI / plugin layer:
 * its boundary for this path is the Python class surface of layers/ (SURVEY.md
 * 8b).  Each entry point below replaces the body of one reference method; the
 * Python host side (pytorch_bayesiancnn_b200/) keeps the reference's class and
 * argument names and calls these through ctypes (see INTEGRATION.md for the
 * stub a maintainer of the reference would add).
 *
 * Conventions
 *   - plain pointers and sizes only; no torch types.  All pointers are DEVICE
 *     pointers unless the name ends in _host.  `cuda_stream` is a cudaStream_t
 *     (CUstream) handle passed as void*; every call is asynchronous on it and
 *     never synchronises, allocates or takes ownership.
 *   - parameters are fp32, reference layout: W_mu/W_rho [Cout, Cin, kh, kw]
 *     (OIHW) or [out, in]; bias_mu/bias_rho [Cout].  Activations are logical
 *     NCHW, contiguous.
 *   - return 0 on success, a negative BBB_E_* code on error;
 *     bbb_last_error() gives the message (thread-local).
 *   - noise: eps pointers NULL  => in-kernel Philox4x32-10 keyed by
 *     (seed, stream_id, flat element index) -- see bbb_philox_normal_fill for
 *     the exact stream definition; non-NULL => that tensor is used (parity mode,
 *     identical eps to the reference's CPU-generator draws).
 */
#ifndef BBB_B200_H_
#define BBB_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BBB_ABI_VERSION 2

enum { BBB_VARIANT_BBB = 0,   /* weight-space sampling   (layers/BBB/...)      */
       BBB_VARIANT_LRT = 1 }; /* local reparameterisation (layers/BBB_LRT/...) */
enum { BBB_DTYPE_F32 = 0, BBB_DTYPE_BF16 = 1 };
enum { BBB_MATH_FP32 = 0,      /* CUDA-core FFMA, IEEE fp32 accumulate          */
       BBB_MATH_BF16_TC = 1,   /* wgmma bf16 x bf16 -> fp32                     */
       BBB_MATH_AUTO = 2,      /* engine picks per layer shape                  */
       BBB_MATH_TF32_TC = 3 }; /* wgmma tf32 x tf32 -> fp32 (operands rounded to tf32, 10-bit mantissa: what the
                                  reference's own GPU conv computes by default, SURVEY D9); per-layer calls only */
enum { BBB_KL_REFERENCE = 0,   /* as executed by the reference: KL(prior||post) */
       BBB_KL_TEXTBOOK = 1 };  /* KL(q||p)                                      */
enum { BBB_ACT_NONE = 0, BBB_ACT_SOFTPLUS = 1, BBB_ACT_RELU = 2 };

enum { BBB_OK = 0, BBB_E_INVALID = -1, BBB_E_UNSUPPORTED = -2, BBB_E_WORKSPACE = -3,
       BBB_E_CUDA = -4 };

/* Geometry + options of one Bayesian layer call.  A linear layer is the
 * degenerate conv: in_h = in_w = kernel = stride = dil = 1, pad = 0,
 * in_channels = in_features, out_channels = out_features, batch = rows. */
typedef struct bbb_layer_desc {
    int32_t batch;
    int32_t in_channels, in_h, in_w;
    int32_t out_channels;
    int32_t kernel_h, kernel_w;
    int32_t stride_h, stride_w;
    int32_t pad_h, pad_w;
    int32_t dil_h, dil_w;
    int32_t variant;        /* BBB_VARIANT_*                                          */
    int32_t sample;         /* 1: stochastic (self.training or sample); 0: mean only */
    int32_t has_bias;
    int32_t act_dtype;      /* BBB_DTYPE_*: dtype of x and y.  BF16: per-layer forward on
                               BBB_MATH_BF16_TC (or AUTO resolving to it) only; act_std,
                               KL and parameters stay fp32; backward takes F32 only     */
    int32_t math;           /* BBB_MATH_*                                             */
    int32_t kl_convention;  /* BBB_KL_*                                               */
    int32_t epilogue_act;   /* BBB_ACT_*: activation fused after the layer (0 = none) */
    int32_t pool_k, pool_s; /* max-pool fused after the activation (0 = none)         */
    int32_t reserved[4];
    float prior_mu, prior_sigma;
} bbb_layer_desc;

/* Per-element Gaussian prior N(mu_p, sigma_p^2) of one layer, for the *_prior entry points below: the KL of each
 * parameter element is taken against its own (mu_p, sigma_p) instead of (desc->prior_mu, desc->prior_sigma) -- a previous
 * task's posterior (variational continual learning), or a prior centred on pretrained weights.  fp32 DEVICE pointers,
 * contiguous, in the layout of W_mu (OIHW / [out, in]) and of bias_mu ([out_channels]).  All four are read only where
 * a KL is computed (kl_out != NULL); noise, MC-sample folds, operand tiles and outputs do not depend on them.
 * sigma_p > 0 (and finite) is the caller's contract: the device does not check it.
 * A prior is all tensors: w_mu and w_sigma are required, b_mu and b_sigma too when the layer has a bias (else
 * BBB_E_INVALID); a caller with a scalar part fills a tensor with it.  prior == NULL is the scalar call of the
 * entry point without _prior (the same kernels, the same bits); a tensor prior filled with desc->prior_mu /
 * desc->prior_sigma gives that call's KL bit for bit (same kernels' summation order). */
typedef struct bbb_prior {
    const float* w_mu;  const float* w_sigma;   /* layout of W_mu (OIHW / [out, in]); sigma > 0 */
    const float* b_mu;  const float* b_sigma;   /* [out_channels]; required iff has_bias      */
} bbb_prior;

/* Pruning mask of one layer, for the same entry points: pass a bbb_masked_prior as their `prior` and OR
 * BBB_PRIOR_MASKED into the call's kl_convention (desc->kl_convention, or the kl_convention argument of the KL calls);
 * without the flag the entry points read a plain bbb_prior, as before.  w_mask / b_mask are one byte per element of
 * W_mu / bias_mu (0 = pruned, 1 = kept; torch.bool storage), DEVICE pointers in the same layouts; b_mask NULL keeps
 * every bias.  A pruned element is a deterministic 0: BBB weight 0 (not mu + eps sigma), LRT mean and variance
 * operands 0; it adds +0.0 to the KL in its own place (every convention, the scalar or the tensor prior), and every
 * backward gives it exactly 0 gradient in mu and rho.  The mask selects, so a pruned element's mu / rho (inf or NaN
 * included) never reach an output.  Noise is drawn as without a mask: a kept element, and an all-ones mask, give the
 * unmasked call's bits.  The mask is read on every call that gets it, not only where a KL is computed.  The four
 * Gaussian pointers of `prior` all NULL (with w_mask set) = the desc's / call's scalar prior, masked.  The Monte-Carlo
 * KL calls (bbb_kl_mc_*) take no mask. */
#define BBB_PRIOR_MASKED 0x100
typedef struct bbb_masked_prior {
    bbb_prior prior;
    const uint8_t* w_mask;                      /* layout of W_mu, 0/1; NULL: no mask          */
    const uint8_t* b_mask;                      /* [out_channels], 0/1; NULL: every bias kept  */
} bbb_masked_prior;

/* Bytes of caller-allocated scratch a forward/KL call on `desc` needs.  The
 * scratch must be zero-filled ONCE when allocated; calls leave it zeroed where
 * that matters (self-resetting counters).  A desc that folds the MC samples of a BBB layer
 * (reserved[1], on bbb_layer_forward_fused or the per-layer forward) needs one operand set per sample. */
size_t bbb_workspace_bytes(const bbb_layer_desc* desc);

/* Replaces BBBConv2d.forward + .kl_loss:
 *   layers/BBB/BBBConv.py:61-83, layers/BBB_LRT/BBBConv.py:62-87.
 * x, y   : [batch, in_channels, H, W] / [batch, out_channels, OH, OW], fp32, or bf16 with act_dtype = BBB_DTYPE_BF16.
 *          bf16 activations need BBB_MATH_BF16_TC (or AUTO resolving to it; BBB_E_UNSUPPORTED on FP32 / TF32_TC): the
 *          kernel multiplies the bf16 x it reads (x^2 of the LRT variance plane is formed from it) and rounds the fp32
 *          output it computes once (round to nearest even) into y.  Tile schedule, accumulation order, noise, folds and
 *          KL are those of the fp32-I/O call, so on a bf16-representable x, y is bf16(y of the fp32-I/O call) bit for bit
 *          and act_std and the KL are equal.
 * kl_out : nullable; the layer's KL scalar (weights + bias) is WRITTEN here.
 * act_std: nullable, LRT only, fp32 shape of y: sqrt(act_var) (BBB_LRT/BBBConv.py:75)
 *          saved for the backward.
 * eps_a  : BBB: W_eps [Cout,Cin,kh,kw]; LRT: activation eps, shape of y.  NULL => Philox.
 * eps_b  : BBB: bias_eps [Cout]; LRT: unused.                             NULL => Philox.
 * Philox element index: BBB: flat OIHW index for W, |W| + c for bias;
 *                       LRT: NHWC-flat index of y, ((b*OH*OW + pixel)*Cout + c), i.e. the
 *                       eps tensor is fill(numel).view(B,OH,OW,C).permute(0,3,1,2) -- four
 *                       consecutive channels share one Philox call in every kernel.
 * stream_base: nullable DEVICE pointer; when set the effective Philox stream is
 *          stream_id + *stream_base, read by the kernel at run time -- this is how a
 *          captured CUDA graph draws fresh noise on every replay (bbb_noise_advance).
 * desc->reserved[1] > 0 folds Monte-Carlo samples into the batch, as on bbb_layer_forward_fused: row (image) b is image
 *          b % reserved[1] of sample s = b / reserved[1], drawn from Philox stream stream_id + s * stride (stride = the
 *          uint64 in reserved[2] (low) / reserved[3] (high)), with the element index of an unfolded call on that image
 *          -- bit-identical to one call per sample.  LRT: the activation noise of row b.  BBB: sample s multiplies by its
 *          own weight draw; needs (reserved[1] * OH * OW) % 128 == 0 and the workspace of the folding desc.  The KL is
 *          computed once, bit-identical to an unfolded call.  Needs sample == 1, in-kernel noise (eps_a / eps_b NULL,
 *          else BBB_E_UNSUPPORTED), batch % reserved[1] == 0 (else BBB_E_INVALID) and a tensor-core math mode (bf16 /
 *          tf32, or auto resolving to one; else BBB_E_UNSUPPORTED).  reserved[] all zero: no fold.  A folded LRT call
 *          can be trained through: act_std is written for every row, and bbb_lrt_noise_grad with the same desc draws
 *          the noise of the backward row by row from the same streams; the weight and input gradients are plain
 *          contractions over all rows (the CUDA-core backward, bbb_conv2d_backward, does not fold).
 * desc->reserved[0] bits 8..30 (BBB_FIRST_IMAGE_*): the FIRST IMAGE, the global index of image 0 of this call (of each
 *          sample block when folded) when a batch is split into row blocks over several calls or ranks
 *          (bbb_mc_exchange_sharded).  LRT: image b draws its activation noise at element index
 *          (((first_image + b)*OH*OW + pixel)*Cout + c) -- what an unsplit call draws at its rows, bit for bit.  Only the
 *          Philox counter moves; x, y, eps_a and act_std stay indexed by the call's own rows.  BBB weight noise does not
 *          depend on rows.  Accepted by every forward, both backwards and the support queries; a negative reserved[0]
 *          or a first image whose last image would pass int32 element counts ((first_image + rows)*OH*OW*Cout, rows =
 *          reserved[1] when folded, else batch) is BBB_E_INVALID.  0 = the batch starts at image 0 (unsplit). */
#define BBB_FIRST_IMAGE_SHIFT 8
#define BBB_FIRST_IMAGE_MASK 0x7fffff00u
int bbb_conv2d_forward(const bbb_layer_desc* desc, const void* x,
                       const float* W_mu, const float* W_rho,
                       const float* bias_mu, const float* bias_rho,
                       void* y, float* kl_out, float* act_std,
                       const float* eps_a, const float* eps_b,
                       uint64_t seed, uint64_t stream_id, const uint64_t* stream_base,
                       void* workspace, size_t workspace_bytes, void* cuda_stream);

/* Replaces BBBLinear.forward + .kl_loss:
 *   layers/BBB/BBBLinear.py:54-76, layers/BBB_LRT/BBBLinear.py:56-79.
 * Same arguments; desc must be the degenerate (1x1) geometry (a BBB fold then needs reserved[1] % 128 == 0). */
int bbb_linear_forward(const bbb_layer_desc* desc, const void* x,
                       const float* W_mu, const float* W_rho,
                       const float* bias_mu, const float* bias_rho,
                       void* y, float* kl_out, float* act_std,
                       const float* eps_a, const float* eps_b,
                       uint64_t seed, uint64_t stream_id, const uint64_t* stream_base,
                       void* workspace, size_t workspace_bytes, void* cuda_stream);

/* bbb_conv2d_forward / bbb_linear_forward with the layer's KL (kl_out) taken against the per-element prior `prior`
 * (bbb_prior; NULL = the scalar call).  y, act_std and every other output are those of the scalar call, unless a
 * mask (bbb_masked_prior) prunes elements. */
int bbb_conv2d_forward_prior(const bbb_layer_desc* desc, const void* x,
                             const float* W_mu, const float* W_rho,
                             const float* bias_mu, const float* bias_rho,
                             void* y, float* kl_out, float* act_std,
                             const float* eps_a, const float* eps_b,
                             uint64_t seed, uint64_t stream_id, const uint64_t* stream_base,
                             void* workspace, size_t workspace_bytes, void* cuda_stream, const bbb_prior* prior);
int bbb_linear_forward_prior(const bbb_layer_desc* desc, const void* x,
                             const float* W_mu, const float* W_rho,
                             const float* bias_mu, const float* bias_rho,
                             void* y, float* kl_out, float* act_std,
                             const float* eps_a, const float* eps_b,
                             uint64_t seed, uint64_t stream_id, const uint64_t* stream_base,
                             void* workspace, size_t workspace_bytes, void* cuda_stream, const bbb_prior* prior);

/* Host-only query (no GPU work, no GPU needed): would bbb_conv2d_forward / bbb_linear_forward accept this desc, its
 * MC-sample fold (reserved[1..3]) and activation dtype included?  Returns BBB_OK or the error code the call would return
 * (bbb_last_error() says why); pointer, external-eps and workspace checks are the call's own.  A bf16 desc gets the
 * answer of the fp32 one on BBB_MATH_BF16_TC and on AUTO resolving to it, BBB_E_UNSUPPORTED otherwise.  The host side
 * asks before it folds a net's samples on the per-layer path, and before it sends a bf16 input as bf16. */
int bbb_forward_supported(const bbb_layer_desc* desc);

/* Activation layouts of the fused tensor-core chain (bbb_layer_forward_fused). */
enum { BBB_LAYOUT_NCHW_F32 = 0,      /* reference layout: [B, C, H, W] fp32                       */
       BBB_LAYOUT_PACKED_BF16 = 1,   /* "tiled packed" bf16: the [B, F] matrix, F = H*W*C, column = (h*W + w)*C + c,
                                        C % 64 == 0, stored as [ceil(B/128)][F/64][128 rows x 128 B] with every 16 KB
                                        block in the K-major SWIZZLE_128B shared-memory image (chunk c of row r at
                                        chunk c ^ (r & 7)); pitch arguments carry F.  When the square is carried too
                                        (LRT consumer) each block is [x | x^2] = 32 KB and x_sq / y_sq = base + 8192 elements */
       BBB_LAYOUT_ROWMAJOR_F32 = 2 };/* [B, OH*OW, Cout] fp32 (logits when OH*OW == 1)            */

/* One Bayesian layer of a fused chain: the layer forward + KL (as bbb_conv2d_forward /
 * bbb_linear_forward) with the model file's activation (desc->epilogue_act) and 2x2/2
 * max-pool (desc->pool_k == 2) fused into the epilogue, reading and writing the packed
 * bf16 inter-layer format so the next layer's operand is a plain 2-D TMA box.  Replaces,
 * per [BBBConv2d|BBBLinear, nn.Softplus|nn.ReLU, nn.MaxPool2d(2,2), FlattenLayer] run of
 * children in ModuleWrapper.forward (layers/misc.py:16-18; BayesianAlexNet.py:34-53).
 *   x, x_sq  : input and (LRT, packed input only) its element-wise square
 *   in_pitch : elements per row of a packed input;  prev_hw: for a linear layer fed by a
 *              flattened HxW map, H*W of that map (reference feature order is c*HW + pix)
 *   y, y_sq  : output and (packed output, nullable) its square for a following LRT layer
 * Forward only (math = BBB_MATH_BF16_TC); eps / Philox / KL semantics as the unfused calls.
 * desc->reserved[0] splits the call so the parameter-only half can run on a side stream, off
 * the activation critical path: BBB_FUSED_PREP_ONLY launches just the weight-prep kernel
 * (sigma, eps, bf16 operand tiles, KL -> kl_out; x/y unused), BBB_FUSED_SKIP_PREP just the GEMM
 * kernel (the caller orders it after the prep, e.g. with an event).  0 = both, in order.  BBB_FUSED_NO_TIMELINE
 * (or'ed in): the call's kernels take no slot of the debug timeline (bbb_debug_set_timeline) -- for launches outside the
 * step being traced, such as operand tiles prepared once per parameter version.  Bits 8..30 of reserved[0]
 * carry the first image of a row block, as on bbb_conv2d_forward (the phase stays in bits 0..2).
 * desc->reserved[1] > 0 folds Monte-Carlo samples into the batch (in-kernel Philox noise only; what
 * uncertainty_estimation.py:38-41 does by repeating the input): row b of the batch is image b % reserved[1] of sample
 * s = b / reserved[1], whose noise comes from Philox stream stream_id + s * stride, stride = the uint64 in reserved[2]
 * (low) / reserved[3] (high) -- bit-identical to separate calls per sample.  LRT: the activation noise of row b.  BBB:
 * sample s multiplies by its own weights and bias, W_mu + softplus(W_rho) * eps with eps drawn from that stream (same
 * element index as an unfolded call); needs reserved[1] % 128 == 0 (else BBB_E_UNSUPPORTED) and batch / reserved[1]
 * times the operand workspace (bbb_workspace_bytes of the folding desc).  Either way the KL is computed once, as by an
 * unfolded call.  The gather path (an NCHW input the stride-4 kernel does not take) does not fold.  The NCHW input of
 * the first layer then holds reserved[1] images (it is not repeated). */
enum { BBB_FUSED_PREP_ONLY = 1, BBB_FUSED_SKIP_PREP = 2, BBB_FUSED_NO_TIMELINE = 4 };
int bbb_layer_forward_fused(const bbb_layer_desc* desc,
                            const void* x, const void* x_sq, int32_t in_layout, int32_t in_pitch, int32_t prev_hw,
                            const float* W_mu, const float* W_rho,
                            const float* bias_mu, const float* bias_rho,
                            void* y, void* y_sq, int32_t out_layout, int32_t out_pitch,
                            float* kl_out, const float* eps_a, const float* eps_b,
                            uint64_t seed, uint64_t stream_id, const uint64_t* stream_base,
                            void* workspace, size_t workspace_bytes, void* cuda_stream);
/* bbb_layer_forward_fused with the KL taken against the per-element prior `prior` (bbb_prior; NULL = the scalar call).
 * Only the weight-prep kernel reads it, a mask (bbb_masked_prior) included (a BBB_FUSED_SKIP_PREP call computes no KL
 * and ignores it: the prepared operands already hold the mask of the prep that wrote them). */
int bbb_layer_forward_fused_prior(const bbb_layer_desc* desc,
                                  const void* x, const void* x_sq, int32_t in_layout, int32_t in_pitch, int32_t prev_hw,
                                  const float* W_mu, const float* W_rho,
                                  const float* bias_mu, const float* bias_rho,
                                  void* y, void* y_sq, int32_t out_layout, int32_t out_pitch,
                                  float* kl_out, const float* eps_a, const float* eps_b,
                                  uint64_t seed, uint64_t stream_id, const uint64_t* stream_base,
                                  void* workspace, size_t workspace_bytes, void* cuda_stream, const bbb_prior* prior);

/* Host-only query (no GPU work, no GPU needed): would bbb_layer_forward_fused accept this layer with these layouts?
 * Returns BBB_OK, or the error code the call would return (bbb_last_error() says why).  The host-side planner
 * (fused.plan) asks before it commits a ModuleWrapper child list to the fused chain. */
int bbb_fused_supported(const bbb_layer_desc* desc, int32_t in_layout, int32_t in_pitch, int32_t prev_hw,
                        int32_t out_layout, int32_t out_pitch);

/* Replaces layer.kl_loss() -> metrics.calculate_kl (metrics.py:27-29 with the call
 * binding of layers/BBB/BBBConv.py:80-82) when no forward preceded it: sigma is
 * recomputed from rho.  n_w = |W|, n_b = |bias| (0 if none). */
int bbb_kl_forward(const float* W_mu, const float* W_rho, uint64_t n_w,
                   const float* bias_mu, const float* bias_rho, uint64_t n_b,
                   float prior_mu, float prior_sigma, int32_t kl_convention,
                   float* kl_out, void* workspace, size_t workspace_bytes, void* cuda_stream);

/* bbb_kl_forward against the per-element prior `prior` (bbb_prior over W_mu's n_w and bias_mu's n_b elements; the
 * bias pointers are required when n_b > 0).  prior_mu / prior_sigma are then not used (unless it is a mask only,
 * bbb_masked_prior); NULL = bbb_kl_forward.  Pruned elements add +0.0 in their place of the same sum. */
int bbb_kl_forward_prior(const float* W_mu, const float* W_rho, uint64_t n_w,
                         const float* bias_mu, const float* bias_rho, uint64_t n_b,
                         float prior_mu, float prior_sigma, int32_t kl_convention,
                         float* kl_out, void* workspace, size_t workspace_bytes, void* cuda_stream,
                         const bbb_prior* prior);

/* d(kl)/d(mu), d(kl)/d(rho), scaled by *grad_kl (device scalar) and ACCUMULATED
 * into g_mu / g_rho (SURVEY.md Appendix A). */
int bbb_kl_backward(const float* mu, const float* rho, uint64_t n,
                    float prior_mu, float prior_sigma, int32_t kl_convention,
                    const float* grad_kl, float* g_mu, float* g_rho, void* cuda_stream);
/* bbb_kl_backward of n elements (a weight tensor, or a bias) against the per-element prior prior->w_mu / prior->w_sigma,
 * laid out like mu (b_mu / b_sigma are not read: for a bias, pass its prior in the w_ fields).  No gradient flows to
 * the prior.  NULL = bbb_kl_backward.  With a mask (bbb_masked_prior; w_mask is the n elements' mask, b_mask is not
 * read) nothing is added to g_mu / g_rho at a pruned element. */
int bbb_kl_backward_prior(const float* mu, const float* rho, uint64_t n,
                          float prior_mu, float prior_sigma, int32_t kl_convention,
                          const float* grad_kl, float* g_mu, float* g_rho, void* cuda_stream,
                          const bbb_prior* prior);

/* The scale-mixture prior of Bayes by Backprop (Blundell et al. 2015, section 3.3; nothing in the reference):
 *   p(w) = pi N(w; 0, sigma1^2) + (1 - pi) N(w; 0, sigma2^2),   usually sigma1 > sigma2: a wide slab and a narrow spike.
 * HOST values.  0 < pi <= 1, sigma1 > 0, sigma2 > 0, all finite and sigma^2 within fp32 range, else BBB_E_INVALID
 * (pi == 1 is the single Gaussian N(0, sigma1^2)). */
typedef struct bbb_mixture_prior { float pi, sigma1, sigma2; } bbb_mixture_prior;

/* Monte-Carlo estimate of KL(q || p) of a layer against a mixture prior, which has no closed form.  For a parameter
 * element with q = N(mu, sigma^2), sigma = log1p(exp(rho)), and one standard normal eps:
 *   w    = mu + sigma eps
 *   term = -log sigma - 1/2
 *          - logsumexp(log pi - log sigma1 - w^2 / (2 sigma1^2), log(1 - pi) - log sigma2 - w^2 / (2 sigma2^2))
 * kl_out[d] = sum of the terms over W, then the bias.  The entropy half is exact and only -E_q[log p] is sampled (the
 * 1/2 log 2 pi of the two halves cancel), so pi == 1 converges to the textbook Gaussian KL.  It is always an estimate of
 * KL(q || p): kl_convention has no meaning here.
 * Noise: draw d uses Philox stream stream_id (+ *stream_base when not NULL, read on the device) + d * draw_stride of
 * `seed`; element i of W draws normal(i) of it and bias element n draws normal(n_w + n), whoever computes it.  Draw d
 * of a call therefore equals, bit for bit, the single-draw call on stream_id + d * draw_stride: with the stride of an
 * MC-sample fold, one call gives the per-sample estimates of the folded samples.  The layer forwards do not compute this
 * term: call them with kl_out == NULL and take the layer's KL from here.
 * workspace: bbb_kl_mc_workspace_bytes(n_draws) bytes, zero-filled once when allocated (self-resetting counters); calls
 * that may run concurrently need workspaces of their own.  n_draws >= 1, else BBB_E_INVALID. */
size_t bbb_kl_mc_workspace_bytes(int32_t n_draws);
int bbb_kl_mc_forward(const float* W_mu, const float* W_rho, uint64_t n_w,
                      const float* bias_mu, const float* bias_rho, uint64_t n_b,
                      const bbb_mixture_prior* prior,
                      uint64_t seed, uint64_t stream_id, const uint64_t* stream_base,
                      int32_t n_draws, uint64_t draw_stride,
                      float* kl_out /* [n_draws] */, void* workspace, size_t workspace_bytes, void* cuda_stream);

/* Reparameterisation gradient of bbb_kl_mc_forward for n elements (a weight tensor with first_element = 0, or the bias
 * with first_element = n_w), eps drawn again from the same streams (element i draws normal(first_element + i)):
 *   s = w (r1 / sigma1^2 + r2 / sigma2^2)   with r1, r2 the softmax of the two logsumexp arguments  (= -d log p / dw)
 *   d/dmu = s     d/dsigma = -1/sigma + s eps     d/drho = sigmoid(rho) d/dsigma
 * g_mu / g_rho are ACCUMULATED into: += sum_d grad_kl[d] * (...), draws in ascending order (grad_kl: n_draws device
 * floats). */
int bbb_kl_mc_backward(const float* mu, const float* rho, uint64_t n, uint64_t first_element,
                       const bbb_mixture_prior* prior,
                       uint64_t seed, uint64_t stream_id, const uint64_t* stream_base,
                       int32_t n_draws, uint64_t draw_stride,
                       const float* grad_kl /* [n_draws] */, float* g_mu, float* g_rho, void* cuda_stream);

/* Backward of bbb_conv2d_forward / bbb_linear_forward (SURVEY.md Appendix A).
 * Regenerates eps from (seed, stream_id) or reads eps_a/eps_b exactly like the
 * forward (the first image of desc->reserved[0] included).  grad_x nullable.  g_* are ACCUMULATED into (caller zeroes).
 * act_std: LRT only, the tensor the forward saved.                            */
int bbb_conv2d_backward(const bbb_layer_desc* desc, const void* x, const void* grad_y,
                        const float* W_mu, const float* W_rho,
                        const float* bias_mu, const float* bias_rho,
                        const float* act_std,
                        const float* eps_a, const float* eps_b,
                        uint64_t seed, uint64_t stream_id, const uint64_t* stream_base,
                        void* grad_x, float* g_W_mu, float* g_W_rho,
                        float* g_bias_mu, float* g_bias_rho,
                        void* workspace, size_t workspace_bytes, void* cuda_stream);
int bbb_linear_backward(const bbb_layer_desc* desc, const void* x, const void* grad_y,
                        const float* W_mu, const float* W_rho,
                        const float* bias_mu, const float* bias_rho,
                        const float* act_std,
                        const float* eps_a, const float* eps_b,
                        uint64_t seed, uint64_t stream_id, const uint64_t* stream_base,
                        void* grad_x, float* g_W_mu, float* g_W_rho,
                        float* g_bias_mu, float* g_bias_rho,
                        void* workspace, size_t workspace_bytes, void* cuda_stream);
/* The same backwards for a layer with a pruning mask (a bbb_masked_prior with BBB_PRIOR_MASKED in desc->kl_convention;
 * its Gaussian pointers are not read here, no KL is involved): a pruned weight is 0 in the input gradient, and nothing
 * is added to g_* at a pruned element.  Two entry points of their own because the backwards above take no prior and
 * their signatures cannot change without breaking their callers; NULL = the call above. */
int bbb_conv2d_backward_prior(const bbb_layer_desc* desc, const void* x, const void* grad_y,
                              const float* W_mu, const float* W_rho,
                              const float* bias_mu, const float* bias_rho,
                              const float* act_std,
                              const float* eps_a, const float* eps_b,
                              uint64_t seed, uint64_t stream_id, const uint64_t* stream_base,
                              void* grad_x, float* g_W_mu, float* g_W_rho,
                              float* g_bias_mu, float* g_bias_rho,
                              void* workspace, size_t workspace_bytes, void* cuda_stream, const bbb_prior* prior);
int bbb_linear_backward_prior(const bbb_layer_desc* desc, const void* x, const void* grad_y,
                              const float* W_mu, const float* W_rho,
                              const float* bias_mu, const float* bias_rho,
                              const float* act_std,
                              const float* eps_a, const float* eps_b,
                              uint64_t seed, uint64_t stream_id, const uint64_t* stream_base,
                              void* grad_x, float* g_W_mu, float* g_W_rho,
                              float* g_bias_mu, float* g_bias_rho,
                              void* workspace, size_t workspace_bytes, void* cuda_stream, const bbb_prior* prior);

/* The engine's noise stream, exposed so the host side of the boundary can draw
 * exactly what a kernel draws: out[i] = N(0,1) lane ((offset+i)&3) of
 * Philox4x32-10(counter = ((offset+i)>>2, stream_id), key = seed), Box-Muller. */
int bbb_philox_normal_fill(float* out, uint64_t n, uint64_t seed, uint64_t stream_id,
                           uint64_t offset, void* cuda_stream);

/* Backward of the LRT noise term (layers/BBB_LRT/BBBConv.py:75-79, BBB_LRT/BBBLinear.py:67-71):
 *   gv = grad_y * eps / (2 * act_std)   element for element, fp32, the shape of y,
 * with eps regenerated exactly as bbb_conv2d_forward / bbb_linear_forward of `desc` drew it:
 * stream stream_id (+ *stream_base when non-NULL, read on the device), NHWC element index, the first image of
 * reserved[0], and with reserved[1..3] the per-row sample streams of an MC-sample fold.  No eps tensor is made.
 * grad_y, act_std (what the forward saved) and gv are NCHW [batch, out_channels, OH, OW] (a linear layer: [batch, out]).
 * The two multiplies and the division are separate IEEE round-to-nearest operations (no FMA, no approximate division),
 * so gv is bit for bit what the three element-wise ops compute on eps = bbb_philox_normal_fill's numbers.
 * Refused: a BBB desc (BBB_E_INVALID), sample == 0 (BBB_E_UNSUPPORTED), batch % reserved[1] != 0 (BBB_E_INVALID), a
 * first image or fold whose counts would pass int32 (BBB_E_INVALID, as the forward). */
int bbb_lrt_noise_grad(const bbb_layer_desc* desc, const float* grad_y, const float* act_std,
                       uint64_t seed, uint64_t stream_id, const uint64_t* stream_base,
                       float* gv, void* cuda_stream);

/* *base += inc on the device (one tiny kernel; put it at the head of a captured
 * graph so each replay moves every layer to a fresh Philox stream). */
int bbb_noise_advance(uint64_t* base, uint64_t inc, void* cuda_stream);

/* One step of a Monte-Carlo engine that keeps steps in flight, enqueued in one host call from the raw handles of its
 * captured graphs (cudaGraphExec_t), streams (cudaStream_t) and events (cudaEvent_t):
 *   run_stream != caller_stream: record in_ready on caller_stream, run_stream waits for it (the caller's work so far);
 *   run_stream waits for wait_a and wait_b (each nullable: e.g. the last exchange that read this step's buffers);
 *   chain_exec launched on run_stream, chain_done recorded there; result_stream waits for chain_done;
 *   exch_exec launched on result_stream, exch_done recorded there.
 * The same work as the runtime calls one by one, without a host round trip per call, so that the host keeps ahead of
 * steps of ~0.1 ms.  Enqueues no kernel of its own. */
int bbb_mc_graph_step(void* caller_stream, void* run_stream, void* in_ready, void* wait_a, void* wait_b,
                      void* chain_exec, void* chain_done, void* result_stream, void* exch_exec, void* exch_done);

/* Monte-Carlo combine that sits directly above the path (main_bayesian.py:46-53,
 * utils.py:14-22): logits [S, B, C] fp32 -> log_outputs [B, C] =
 * logmeanexp_s(log_softmax(logits[s])).  Also emits per-sample partials
 * (sum_s softmax, sum_s softmax^2, sum_s logits) [3, B, C] if `moments` != NULL
 * (uncertainty_estimation.py:70-96).  These are raw sums: sum p^2 / S - (sum p / S)^2
 * cancels when the samples agree and is no way to get the epistemic variance (the
 * exchange below returns it centred).  A class at -inf in some samples adds nothing
 * to log_outputs for those samples. */
int bbb_mc_combine(const float* logits, int32_t S, int32_t B, int32_t C,
                   float* log_outputs, float* moments, void* cuda_stream);

/* Monte-Carlo combine + ELBO head + uncertainty outputs, FUSED with the one exchange of the forward path
 * (main_bayesian.py:46-61, utils.py:14-22, metrics.py:12-14,23-24, uncertainty_estimation.py:70-96; SURVEY.md 8e, f3, f4).
 * The num_ens samples are sharded over `world` ranks (one process per GPU); this rank holds `S_local` of the
 * `S_total` samples' logits [S_local, B, C].  One kernel: per-(image, class) partials of the local samples
 * (the exact (max, sum-exp) pair of logmeanexp, + mean p / M2 = sum (p - mean)^2 / sum logits and the sample count with
 * BBB_MC_MOMENTS, the ranks' moments merged with Chan's update) are stored straight
 * into every rank's receive buffer over NVLink (peer-mapped memory, below) as 8-byte words {value, sequence number};
 * the receiver polls each word until its tag matches (no fence, no flag; a lost peer is a counted time-out, never a
 * hang) and the result is finished locally in fixed rank order (bitwise identical on all ranks):
 *   log_outputs [B,C] = logmeanexp_j log_softmax(logits_j)      kl_out = sum_j kl_j / S_total
 *   pred / epistemic / aleatoric [B,C], entropy [B]             (nullable; need BBB_MC_MOMENTS)
 *     epistemic = mean_s (p_hat_s - p_bar)^2 >= 0 (centred), aleatoric = p_bar (1 - p_bar) - epistemic
 *   head [4] = {nll*train_size + beta*kl, nll, accuracy, beta*kl}   (nullable; needs labels [B] int64)
 * BBB_MC_NORMALIZED: p_hat = softplus(logits) / sum softplus (uncertainty_estimation.py:73-75) instead of softmax.
 * peer_buffers: HOST array of `world` device pointers, one receive buffer per rank (bbb_mc_buffer_bytes each, zero-
 *   filled once; [rank] is the local one; with world == 1 any device allocation will do);
 * state: local device scratch of bbb_mc_state_bytes(), zero-filled once.  Sequence numbers inside make the buffers
 * reusable call after call (and CUDA-graph replay after replay) with no reset.  Every rank must make the same calls.
 * kl: n_kl device floats whose SUM is one sample's KL (e.g. the per-layer scalars the layer calls wrote: the sum over
 *   layers of ModuleWrapper.forward, layers/misc.py:21-23, happens here); n_kl <= 0 means 1.
 * noise_base (nullable): *noise_base += noise_inc when the launch has finished -- the last kernel of a captured step
 *   moves the Philox stream base for the next replay (replaces a leading bbb_noise_advance launch).
 * BBB_MC_INFO (needs BBB_MC_MOMENTS; see bbb_mc_exchange_info) adds one [B] plane per rank to the receive buffer:
 *   bbb_mc_buffer_bytes grows only when the flag is set, and returns 0 for BBB_MC_INFO without BBB_MC_MOMENTS. */
enum { BBB_MC_MOMENTS = 1, BBB_MC_NORMALIZED = 2, BBB_MC_INFO = 4 };
size_t bbb_mc_buffer_bytes(int32_t B, int32_t C, int32_t flags, int32_t world);
size_t bbb_mc_state_bytes(void);
int bbb_mc_exchange(const float* logits, int32_t S_local, int32_t S_total, int32_t B, int32_t C, const float* kl,
                    int32_t n_kl, int32_t flags, const int64_t* labels, float train_size, float beta, int32_t rank,
                    int32_t world, void* const* peer_buffers, void* state, float* log_outputs, float* kl_out, float* pred,
                    float* epistemic, float* aleatoric, float* entropy, float* head, uint64_t* noise_base,
                    uint64_t noise_inc, void* cuda_stream);
/* bbb_mc_exchange plus the rest of the entropy decomposition  H[p_bar] = E_s H[p_hat_s] + I(y; w)  (total = expected
 * entropy, the aleatoric part + mutual information / BALD, the epistemic part), for each image b:
 *   p_hat_s            the per-sample probabilities the moments use: softmax(logits_s), or with BBB_MC_NORMALIZED
 *                      softplus(logits_s) / sum softplus (uncertainty_estimation.py:73-77)
 *   H[p]               = -sum_c p_c log p_c with 0 log 0 = 0 (a class whose probability underflows to 0 adds nothing)
 *   expected_entropy[b] = (1/S_total) sum_{s over all ranks} H[p_hat_s]
 *   mutual_info[b]     = entropy[b] - expected_entropy[b], in fp32 and NOT clamped: rounding may leave it slightly
 *                        negative where the samples agree
 * expected_entropy / mutual_info: [B] fp32 each, nullable.  They need flags & BBB_MC_INFO, which needs
 * BBB_MC_MOMENTS (H[p_bar] comes from the sum-p plane); otherwise BBB_E_INVALID.  Each rank pushes one more word per
 * image (the sum of H[p_hat_s] over its samples; 0 without samples); the sums are finished in rank order, so the outputs
 * are bitwise identical on every rank.  Without BBB_MC_INFO this is bbb_mc_exchange: the same kernel and results. */
int bbb_mc_exchange_info(const float* logits, int32_t S_local, int32_t S_total, int32_t B, int32_t C, const float* kl,
                         int32_t n_kl, int32_t flags, const int64_t* labels, float train_size, float beta, int32_t rank,
                         int32_t world, void* const* peer_buffers, void* state, float* log_outputs, float* kl_out,
                         float* pred, float* epistemic, float* aleatoric, float* entropy, float* head,
                         uint64_t* noise_base, uint64_t noise_inc, float* expected_entropy, float* mutual_info,
                         void* cuda_stream);
/* bbb_mc_exchange_info with the batch split into row blocks as well as the samples into groups, so that every rank works
 * when there are fewer samples than ranks (or they do not divide evenly).  world = Rs x Rb, Rb = batch_shards (world %
 * batch_shards != 0 or batch_shards > B: BBB_E_INVALID).  Rank r is sample group g = r % Rs (it holds the samples
 * {j : j mod Rs == g}) and row block k = r / Rs: images [b0, b1), the blocks as equal as possible, the first B % Rb one
 * image longer.  logits: [S_local, b1 - b0, C] (its rows only); labels: all [B].  Every rank returns the same full
 * [B, C] / [B] outputs and head as bbb_mc_exchange_info, and they are bitwise equal to that call on Rs ranks holding
 * the same samples: the receive buffer is [2 slots][Rs][...] -- bbb_mc_buffer_bytes(B, C, flags, Rs) -- rank (g, k)
 * pushes the words of its rows into slot g of every peer, the block-0 rank of each group its KL word, and the Rs groups
 * are merged in ascending order.  peer_buffers still holds all `world` buffers.  batch_shards == 1 is
 * bbb_mc_exchange_info (the same kernel).  The callers' layer calls draw the rows of a block with the first image b0
 * (desc->reserved[0]), so per-sample logits do not depend on (Rs, Rb). */
int bbb_mc_exchange_sharded(const float* logits, int32_t S_local, int32_t S_total, int32_t B, int32_t C, const float* kl,
                            int32_t n_kl, int32_t flags, const int64_t* labels, float train_size, float beta,
                            int32_t rank, int32_t world, void* const* peer_buffers, void* state, float* log_outputs,
                            float* kl_out, float* pred, float* epistemic, float* aleatoric, float* entropy, float* head,
                            uint64_t* noise_base, uint64_t noise_inc, float* expected_entropy, float* mutual_info,
                            int32_t batch_shards, void* cuda_stream);

/* bbb_mc_exchange_sharded that also adds the step to an evaluation accumulator: validate_model's two numbers
 * (main_bayesian.py:65-86) and calibration over a whole held-out set, with no host read per batch.  batch_shards == 1 is
 * the sample-only split.  Every output of bbb_mc_exchange_sharded is bitwise the same.  Per image b, on the predictive
 * distribution p_bar = exp(log_outputs[b]) (the mean of the per-sample p_hat_s, softmax or softplus-normalised):
 *   conf = p_bar[argmax], correct = (argmax == y) (the first maximal class), nll = -log_outputs[b, y],
 *   brier = sum_c (p_bar_c - [c == y])^2, calibration bin m = clamp(ceil(conf * BBB_MC_CAL_BINS) - 1, 0, BINS - 1):
 *   BBB_MC_CAL_BINS equal-width bins (m / BINS, (m + 1) / BINS] (Guo et al. 2017).
 * metrics: device float64 words, bbb_mc_metrics_bytes() in all, zero-filled by the caller before the first step.  Each
 * launch adds one step (BINS = BBB_MC_CAL_BINS):
 *   [0] steps   [1] images   [2] sum_steps nll_step   [3] sum_steps acc_step   (the per-batch means of the head, fp64)
 *   [4] sum_steps klsum_step, klsum = sum_j kl_j over the S_total samples, NOT divided by S_total (validate_model's kl)
 *   [5] sum nll   [6] sum correct   [7] sum brier                               (over images)
 *   [8 + m] count   [8 + BINS + m] sum conf   [8 + 2 BINS + m] sum correct      (images of bin m)
 * The words behind [8 + 3 BINS] are per-launch scratch.  A loss with a per-batch beta_i is (train_size * [2] +
 * (sum_i beta_i) * [4] / [0]) / [0]: the KL does not depend on the batch.  Sums are taken per warp, per CTA and over the
 * CTAs in a fixed order, in double precision: the accumulator is bitwise the same on every rank and from run to run.
 * Launches that share an accumulator must run one after another (e.g. on one stream); engines of different batch sizes
 * may share one.  metrics == NULL or labels == NULL: BBB_E_INVALID. */
enum { BBB_MC_CAL_BINS = 15 };
size_t bbb_mc_metrics_bytes(void);
int bbb_mc_exchange_metrics(const float* logits, int32_t S_local, int32_t S_total, int32_t B, int32_t C, const float* kl,
                            int32_t n_kl, int32_t flags, const int64_t* labels, float train_size, float beta,
                            int32_t rank, int32_t world, void* const* peer_buffers, void* state, float* log_outputs,
                            float* kl_out, float* pred, float* epistemic, float* aleatoric, float* entropy, float* head,
                            uint64_t* noise_base, uint64_t noise_inc, float* expected_entropy, float* mutual_info,
                            int32_t batch_shards, double* metrics, void* cuda_stream);

/* Peer-mapped receive buffers for bbb_mc_exchange (one process per GPU, same node): allocate locally, export a
 * 64-byte CUDA-IPC handle, ship it to the peers by any host channel (the Python side uses torch.distributed),
 * import theirs.  These five calls are the only ones in this library that allocate or synchronise. */
int bbb_comm_alloc(size_t bytes, void** dev_ptr);            /* cudaMalloc + zero fill                 */
int bbb_comm_free(void* dev_ptr);
int bbb_comm_export(void* dev_ptr, void* handle64_host);     /* writes 64 bytes                        */
int bbb_comm_import(const void* handle64_host, void** peer_ptr);
int bbb_comm_unimport(void* peer_ptr);

const char* bbb_last_error(void);
int32_t bbb_abi_version(void);
/* Number of kernels this library has launched since load (all entry points). */
uint64_t bbb_launch_count(void);
/* Tile policy of the fused chain's tap-GEMM layers (bbb_layer_forward_fused), read at launch (= graph capture) time:
 * 0 (default) = 128-column tiles only where the grid still covers most of the SMs (best latency of ONE step);
 * 1 = 128-column tiles wherever Cout allows (fewer operand bytes per MAC; best throughput when several independent
 * steps are in flight and fill the SMs a narrow grid leaves idle; slower for a single step).  Returns the previous
 * value. */
int32_t bbb_set_wide_tiles(int32_t prefer_wide);

#ifdef __cplusplus
}
#endif
#endif  /* BBB_B200_H_ */
