// C-ABI entry points of libbbb_b200.so (declared in include/bbb_b200.h).
#include <atomic>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>

#include "common.cuh"
#include "fwd_simt.cuh"
#include "misc_kernels.cuh"
#include "kl_mc.cuh"
#include "bwd_simt.cuh"
#include "fwd_tc.cuh"
#include "fused_tc.cuh"
#include "conv_s4_tc.cuh"
#include "mc_head.cuh"

namespace {

thread_local char g_err[512] = "";
std::atomic<uint64_t> g_launches{0};
std::atomic<int> g_wide_tiles{0};   // bbb_set_wide_tiles
long long* g_trace = nullptr;      // debug hook (bbb_debug_set_trace)
long long* g_mcx_trace = nullptr;  // debug hook (bbb_debug_set_mcx_trace): handshake stamps of the exchange kernel
// debug hook (bbb_debug_set_timeline): launch k of the instrumented kernels writes [first CTA entry, last CTA
// exit] in %globaltimer ns to g_tl[2k], g_tl[2k+1]; the slot index is fixed at launch (= capture) time
long long* g_tl = nullptr;
int g_tl_cap = 0, g_tl_n = 0;
char g_tl_names[256][64];
long long* tl_slot(bool used, const char* kind, const bbb::Geom& g) {
    if (!g_tl || !used || g_tl_n >= g_tl_cap || g_tl_n >= 256) return nullptr;
    snprintf(g_tl_names[g_tl_n], sizeof(g_tl_names[0]), "%s M=%d N=%d K=%d", kind, g.M, g.N, g.K);
    return g_tl + 4 * (g_tl_n++);
}

int fail(int code, const char* fmt, ...) {
    va_list ap; va_start(ap, fmt); vsnprintf(g_err, sizeof(g_err), fmt, ap); va_end(ap);
    return code;
}
int cuda_fail(cudaError_t e, const char* what) {
    return fail(BBB_E_CUDA, "%s: %s", what, cudaGetErrorString(e));
}

constexpr size_t kCounterBytes = 64;
constexpr size_t kMaxKlSlots = 4096;
constexpr size_t kBaseWorkspace = kCounterBytes + kMaxKlSlots * sizeof(double);
constexpr size_t kTcOffset = (kBaseWorkspace + 1023) / 1024 * 1024;   // prepared-operand region (tensor-core path)

int sm_count() {
    static int n = 0;
    if (n == 0) {
        int dev = 0; cudaGetDevice(&dev);
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    }
    return n;
}

// Bytes of one set of prepared operands (tiles, zero sub-tile, bias rows) of whichever tensor-core path takes the layer.
size_t tc_set_bytes(const bbb::Geom& g) {
    return std::max({bbb::tc_workspace_bytes(g), bbb::fused_workspace_bytes(g), bbb::conv_s4_workspace_bytes(g)});
}
// Operand sets a call prepares: batch / rows for a BBB fold (one weight draw per MC sample), else 1.
int weight_sets(const bbb_layer_desc& d, const bbb::Geom& g) {
    const int rows = d.reserved[1];
    return (d.variant == BBB_VARIANT_BBB && rows > 0 && g.B % rows == 0) ? g.B / rows : 1;
}
size_t set_stride(const bbb::Geom& g) { return (tc_set_bytes(g) + 1023) / 1024 * 1024; }

bool s4_enabled() {
    static const bool on = [] { const char* e = getenv("BBB_B200_CONV1_DIRECT"); return !(e && e[0] == '0'); }();
    return on;
}

int first_image_of(const bbb_layer_desc& d) { return (int)(((uint32_t)d.reserved[0] & BBB_FIRST_IMAGE_MASK) >> BBB_FIRST_IMAGE_SHIFT); }

int check_desc(const bbb_layer_desc* d, bbb::Geom& g, bool linear) {
    if (!d) return fail(BBB_E_INVALID, "desc is NULL");
    if (!bbb::make_geom(*d, g)) return fail(BBB_E_INVALID, "invalid layer geometry");
    if (linear && !g.linear_like) return fail(BBB_E_INVALID, "bbb_linear_*: desc is not the degenerate 1x1 geometry");
    if (d->variant != BBB_VARIANT_BBB && d->variant != BBB_VARIANT_LRT) return fail(BBB_E_INVALID, "bad variant %d", d->variant);
    if (d->kl_convention != BBB_KL_REFERENCE && d->kl_convention != BBB_KL_TEXTBOOK) return fail(BBB_E_INVALID, "bad kl_convention");
    if (d->epilogue_act < BBB_ACT_NONE || d->epilogue_act > BBB_ACT_RELU) return fail(BBB_E_INVALID, "bad epilogue_act");
    if (!(d->prior_sigma > 0.0f)) return fail(BBB_E_INVALID, "prior_sigma must be > 0");
    // first image of a row block (reserved[0] bits 8..30, include/bbb_b200.h): the noise index of its last image must
    // still be an int32 element count, as that of an unsplit batch is
    if (d->reserved[0] < 0) return fail(BBB_E_INVALID, "negative first image (desc->reserved[0] = %d)", d->reserved[0]);
    const long images = (long)first_image_of(*d) + (d->reserved[1] > 0 ? d->reserved[1] : g.B);
    if (images * g.OHW * g.N > 0x7fffffffL)
        return fail(BBB_E_INVALID, "first image %d: image %ld x %d x %d outputs passes int32 element counts",
                    first_image_of(*d), images, g.OHW, g.N);
    return BBB_OK;
}

// Pool, math-mode and shape checks of the per-layer forward (host logic only); `math` = the resolved BBB_MATH_*.
int layer_math(const bbb_layer_desc* d, const bbb::Geom& g, int& math) {
    if (d->pool_k != 0) return fail(BBB_E_UNSUPPORTED, "fused max-pool epilogue is not available on this path");
    if (d->act_dtype != BBB_DTYPE_F32 && d->act_dtype != BBB_DTYPE_BF16) return fail(BBB_E_UNSUPPORTED, "bad act_dtype %d", d->act_dtype);
    math = d->math;
    if (math == BBB_MATH_AUTO) math = bbb::tc_supported(g) ? BBB_MATH_BF16_TC : BBB_MATH_FP32;
    if (math == BBB_MATH_BF16_TC || math == BBB_MATH_TF32_TC) {
        if (!bbb::tc_supported(g)) return fail(BBB_E_UNSUPPORTED, "tensor-core math mode: shape not supported by the tensor-core path");
        if (math == BBB_MATH_TF32_TC && d->act_dtype != BBB_DTYPE_F32)
            return fail(BBB_E_UNSUPPORTED, "bf16 activations take bf16 operands (BBB_MATH_BF16_TC), not tf32");
        return BBB_OK;
    }
    if (math != BBB_MATH_FP32) return fail(BBB_E_INVALID, "bad math mode %d", d->math);
    if (d->act_dtype != BBB_DTYPE_F32) return fail(BBB_E_UNSUPPORTED, "BBB_MATH_FP32 path takes fp32 activations only");
    if ((size_t)bbb::simt_kl_slots(g) > kMaxKlSlots || bbb::simt_kl_slots(g) > 65535)
        return fail(BBB_E_UNSUPPORTED, "out_channels too large for the CUDA-core path (%d column tiles)", bbb::simt_kl_slots(g));
    return BBB_OK;
}

// MC-sample fold checks of the per-layer forward (desc->reserved[1..3], include/bbb_b200.h); a no-op when reserved[1] == 0
int layer_fold_check(const bbb_layer_desc* d, const bbb::Geom& g, int math) {
    const int rows = d->reserved[1];
    if (rows <= 0) return BBB_OK;
    if (!d->sample) return fail(BBB_E_UNSUPPORTED, "MC-sample folding needs a sampling call");
    if (g.B % rows) return fail(BBB_E_INVALID, "batch %d is not a multiple of the rows per MC sample %d", g.B, rows);
    if (math == BBB_MATH_FP32) return fail(BBB_E_UNSUPPORTED, "MC-sample folding needs a tensor-core math mode");
    // a 128-row GEMM tile multiplies by ONE weight sample's operand set
    if (d->variant == BBB_VARIANT_BBB && ((long)rows * g.OHW) % bbb::TC_BM)
        return fail(BBB_E_UNSUPPORTED, "BBB MC-sample folding needs rows x OH x OW %% %d == 0 (got %d x %d)", bbb::TC_BM, rows, g.OHW);
    return BBB_OK;
}

// The MC-sample fold of a tensor-core call (desc->reserved[1..3], include/bbb_b200.h; rows = 0: none).  A fold draws its
// noise in-kernel, so it takes no external eps.
int layer_fold(const bbb_layer_desc* d, const bbb::Geom& g, const float* eps_a, const float* eps_b, bbb::McFold& fold) {
    fold.rows = 0; fold.stride = 0; fold.sets = 1; fold.set_bytes = 0;
    fold.first_image = first_image_of(*d);
    if (d->reserved[1] <= 0) return BBB_OK;
    if (eps_a || eps_b) return fail(BBB_E_UNSUPPORTED, "MC-sample folding draws its noise in-kernel (no external eps)");
    fold.rows = d->reserved[1];
    fold.stride = ((unsigned long long)(uint32_t)d->reserved[3] << 32) | (uint32_t)d->reserved[2];
    fold.sets = weight_sets(*d, g);
    fold.set_bytes = set_stride(g);
    return BBB_OK;
}

// The parameter half of a tensor-core call: desc, parameters, noise, KL workspace, operand region (tiles at kTcOffset,
// bias rows `bias_offset` bytes behind them), fold and debug slots.  The timeline slots are taken in launch order.
void layer_args(bbb::LayerArgs& a, const bbb_layer_desc* d, const bbb::Geom& g, const float* W_mu, const float* W_rho,
                const float* bias_mu, const float* bias_rho, float* kl_out, const float* eps_a, const float* eps_b,
                uint64_t seed, uint64_t stream_id, const uint64_t* stream_base, void* ws, size_t bias_offset,
                const bbb::McFold& fold, const char* prep_name, bool do_prep, const char* gemm_name, bool do_gemm) {
    a.g = g; a.w_mu = W_mu; a.w_rho = W_rho; a.b_mu = bias_mu; a.b_rho = bias_rho; a.eps_a = eps_a; a.eps_b = eps_b;
    a.key = bbb::make_key(seed, stream_id); a.stream_base = (const unsigned long long*)stream_base;
    a.kl_counter = (unsigned int*)ws; a.kl_partials = (double*)((char*)ws + kCounterBytes); a.kl_out = kl_out;
    a.prior_mu = d->prior_mu; a.prior_sigma = d->prior_sigma;
    a.sample = d->sample; a.kl_convention = d->kl_convention; a.has_bias = d->has_bias; a.act = d->epilogue_act;
    a.variant = d->variant;
    a.wtiles = (__nv_bfloat16*)((char*)ws + kTcOffset);
    a.bias_ws = (float*)((char*)ws + kTcOffset + bias_offset);
    a.fold = fold;
    a.trace = g_trace;
    a.tl_prep = tl_slot(do_prep, prep_name, g);
    a.tl_gemm = tl_slot(do_gemm, gemm_name, g);
}

// The pruning mask of a call (bbb_masked_prior): BBB_PRIOR_MASKED in its kl_convention says that `prior` points at a
// bbb_masked_prior.  take_masks clears the flag and returns the masks (NULL without).
struct Masks { const uint8_t* w; const uint8_t* b; };
Masks take_masks(const bbb_prior* prior, int32_t& conv) {
    Masks m = {nullptr, nullptr};
    if (conv & BBB_PRIOR_MASKED) {
        conv &= ~BBB_PRIOR_MASKED;
        if (prior) {
            const bbb_masked_prior* q = reinterpret_cast<const bbb_masked_prior*>(prior);
            m.w = q->w_mask; m.b = q->w_mask ? q->b_mask : nullptr;
        }
    }
    return m;
}
// The same for a call with a desc: the desc without the flag (a copy in `copy` when it had it)
const bbb_layer_desc* desc_masks(const bbb_layer_desc* d, const bbb_prior* prior, bbb_layer_desc& copy, Masks& m) {
    m = Masks{nullptr, nullptr};
    if (!d || !(d->kl_convention & BBB_PRIOR_MASKED)) return d;
    copy = *d;
    m = take_masks(prior, copy.kl_convention);
    return &copy;
}

// A tensor prior (bbb_prior) is all tensors: the weight part always, the bias part with a bias.  All four NULL is the
// scalar prior of the desc / call, valid only beside a mask.
int check_prior(const bbb_prior* q, bool has_bias, const Masks& mk = Masks{nullptr, nullptr}) {
    if (!q) return BBB_OK;
    if (!q->w_mu && !q->w_sigma && !q->b_mu && !q->b_sigma && mk.w) return BBB_OK;
    if (!q->w_mu || !q->w_sigma) return fail(BBB_E_INVALID, "prior: w_mu / w_sigma NULL (a prior is all tensors)");
    if (has_bias && (!q->b_mu || !q->b_sigma)) return fail(BBB_E_INVALID, "prior: has_bias set but b_mu / b_sigma NULL");
    return BBB_OK;
}
// What the kernels get of a tensor prior: its pointers when the call computes a KL, else none (the scalar kernels run
// and nothing of the prior is read); and the mask, always (NULL: the unmasked kernels run)
bbb::PriorPtrs prior_ptrs(const bbb_prior* q, const float* kl_out, const Masks& mk = Masks{nullptr, nullptr}) {
    bbb::PriorPtrs t = {nullptr, nullptr, nullptr, nullptr, mk.w, mk.b};
    if (q && kl_out) { t.w_mu = q->w_mu; t.w_sigma = q->w_sigma; t.b_mu = q->b_mu; t.b_sigma = q->b_sigma; }
    return t;
}

// Counters of a Monte-Carlo KL call (one per draw), padded so that the partial rows behind them stay aligned.
size_t kl_mc_counter_bytes(size_t n_draws) { return (n_draws * sizeof(unsigned int) + 255) / 256 * 256; }

// The scale-mixture prior of a Monte-Carlo KL call comes from outside the library: 0 < pi <= 1, sigma1, sigma2 > 0, all
// finite, and sigma^2 within fp32 range (1 / (2 sigma^2) is what the kernels multiply by).
int check_mixture(const bbb_mixture_prior* p, int32_t n_draws, bbb::MixPrior& q) {
    if (!p) return fail(BBB_E_INVALID, "mixture prior is NULL");
    if (!(p->pi > 0.0f && p->pi <= 1.0f)) return fail(BBB_E_INVALID, "mixture prior: pi must be in (0, 1] (got %g)", (double)p->pi);
    if (!(p->sigma1 > 0.0f && std::isfinite(p->sigma1) && p->sigma2 > 0.0f && std::isfinite(p->sigma2)))
        return fail(BBB_E_INVALID, "mixture prior: sigma1 and sigma2 must be finite and > 0 (got %g, %g)", (double)p->sigma1, (double)p->sigma2);
    if (n_draws < 1) return fail(BBB_E_INVALID, "n_draws must be >= 1 (got %d)", n_draws);
    const double s1 = p->sigma1, s2 = p->sigma2, pi = p->pi;
    q.lc1 = (float)(std::log(pi) - std::log(s1));
    q.lc2 = pi < 1.0 ? (float)(std::log1p(-pi) - std::log(s2)) : -INFINITY;
    q.h1 = (float)(0.5 / (s1 * s1));
    q.h2 = (float)(0.5 / (s2 * s2));
    if (!std::isfinite(q.h1) || !std::isfinite(q.h2) || q.h1 == 0.0f || q.h2 == 0.0f)
        return fail(BBB_E_INVALID, "mixture prior: sigma^2 outside fp32 range (got %g, %g)", s1, s2);
    return BBB_OK;
}

int forward_impl(const bbb_layer_desc* d, bool linear, const void* x, const float* W_mu, const float* W_rho,
                 const float* bias_mu, const float* bias_rho, void* y, float* kl_out, float* act_std,
                 const float* eps_a, const float* eps_b, uint64_t seed, uint64_t stream_id, const uint64_t* stream_base, void* ws,
                 size_t ws_bytes, void* stream, const bbb_prior* prior) {
    bbb_layer_desc dcopy;
    Masks mk;
    d = desc_masks(d, prior, dcopy, mk);
    bbb::Geom g;
    if (int rc = check_desc(d, g, linear)) return rc;
    if (!x || !W_mu || !W_rho || !y) return fail(BBB_E_INVALID, "NULL tensor pointer");
    if (d->has_bias && (!bias_mu || !bias_rho)) return fail(BBB_E_INVALID, "has_bias set but bias pointers NULL");
    if (int rc = check_prior(prior, d->has_bias != 0, mk)) return rc;
    if (kl_out && (!ws || ws_bytes < bbb_workspace_bytes(d)))
        return fail(BBB_E_WORKSPACE, "workspace too small: need %zu bytes", bbb_workspace_bytes(d));
    cudaStream_t st = (cudaStream_t)stream;

    int math = BBB_MATH_FP32;
    if (int rc = layer_math(d, g, math)) return rc;
    if (int rc = layer_fold_check(d, g, math)) return rc;
    bbb::McFold fold;
    if (int rc = layer_fold(d, g, eps_a, eps_b, fold)) return rc;
    if (math == BBB_MATH_BF16_TC || math == BBB_MATH_TF32_TC) {
        const size_t need = fold.sets > 1 ? bbb_workspace_bytes(d) : kTcOffset + bbb::tc_workspace_bytes(g);
        if (!ws || ws_bytes < need) return fail(BBB_E_WORKSPACE, "workspace too small for the tensor-core path: need %zu bytes", need);
        const bool tf32 = math == BBB_MATH_TF32_TC;
        bbb::TcArgs a;
        layer_args(a, d, g, W_mu, W_rho, bias_mu, bias_rho, kl_out, eps_a, eps_b, seed, stream_id, stream_base, ws,
                   bbb::tc_bias_offset(g, tf32), fold, "weight_prep", true, "gemm_tc", true);
        a.tf32 = tf32;
        a.skip_prep = 0; a.prep_only = 0; a.y_sq = nullptr; a.out_mode = 2; a.out_pitch = 0; a.pool = 0;
        a.x = x; a.y = y; a.act_std = act_std; a.act_dtype = d->act_dtype;
        int nl = 0;
        cudaError_t e = bbb::launch_fwd_tc(a, st, sm_count(), &nl, prior_ptrs(prior, kl_out, mk));
        if (e != cudaSuccess) return cuda_fail(e, "fwd_tc launch");
        g_launches += nl;
        return BBB_OK;
    }

    bbb::FwdArgs a;
    a.g = g; a.x = (const float*)x; a.w_mu = W_mu; a.w_rho = W_rho; a.b_mu = bias_mu; a.b_rho = bias_rho;
    a.y = (float*)y; a.kl_out = kl_out; a.act_std = act_std; a.eps_a = eps_a; a.eps_b = eps_b;
    a.key = bbb::make_key(seed, stream_id); a.stream_base = (const unsigned long long*)stream_base;
    a.kl_counter = (unsigned int*)ws; a.kl_partials = (double*)((char*)ws + kCounterBytes);
    a.prior_mu = d->prior_mu; a.prior_sigma = d->prior_sigma;
    a.sample = d->sample; a.kl_convention = d->kl_convention; a.has_bias = d->has_bias; a.act = d->epilogue_act;
    a.first_image = first_image_of(*d);
    a.prior = prior_ptrs(prior, kl_out, mk);
    cudaError_t e = d->variant == BBB_VARIANT_LRT ? bbb::launch_fwd_simt<BBB_VARIANT_LRT>(a, st)
                                                  : bbb::launch_fwd_simt<BBB_VARIANT_BBB>(a, st);
    if (e != cudaSuccess) return cuda_fail(e, "fwd_simt launch");
    g_launches += 1;
    return BBB_OK;
}

int backward_impl(const bbb_layer_desc* d, bool linear, const void* x, const void* grad_y, const float* W_mu,
                  const float* W_rho, const float* bias_mu, const float* bias_rho, const float* act_std,
                  const float* eps_a, const float* eps_b, uint64_t seed, uint64_t stream_id, const uint64_t* stream_base, void* grad_x,
                  float* g_W_mu, float* g_W_rho, float* g_bias_mu, float* g_bias_rho, void* ws, size_t ws_bytes,
                  void* stream, const bbb_prior* prior) {
    bbb_layer_desc dcopy;
    Masks mk;
    d = desc_masks(d, prior, dcopy, mk);
    bbb::Geom g;
    if (int rc = check_desc(d, g, linear)) return rc;
    if (!x || !grad_y || !W_mu || !W_rho) return fail(BBB_E_INVALID, "NULL tensor pointer");
    if (d->act_dtype != BBB_DTYPE_F32) return fail(BBB_E_UNSUPPORTED, "backward takes fp32 activations only");
    if (d->epilogue_act != BBB_ACT_NONE || d->pool_k != 0)
        return fail(BBB_E_UNSUPPORTED, "backward through a fused activation/pool epilogue is not available");
    if (d->variant == BBB_VARIANT_LRT && d->sample && !act_std)
        return fail(BBB_E_INVALID, "LRT backward needs the act_std tensor saved by the forward");
    if (int rc = check_prior(prior, d->has_bias != 0, mk)) return rc;
    (void)ws; (void)ws_bytes;
    bbb::BwdArgs a;
    a.g = g; a.x = (const float*)x; a.gy = (const float*)grad_y; a.w_mu = W_mu; a.w_rho = W_rho;
    a.b_mu = bias_mu; a.b_rho = bias_rho; a.act_std = act_std; a.eps_a = eps_a; a.eps_b = eps_b;
    a.key = bbb::make_key(seed, stream_id); a.stream_base = (const unsigned long long*)stream_base;
    a.gx = (float*)grad_x; a.g_w_mu = g_W_mu; a.g_w_rho = g_W_rho; a.g_b_mu = g_bias_mu; a.g_b_rho = g_bias_rho;
    a.sample = d->sample; a.has_bias = d->has_bias; a.variant = d->variant;
    a.first_image = first_image_of(*d);
    a.prior = prior_ptrs(prior, nullptr, mk);       // the backward reads the mask only
    int nl = 0;
    cudaError_t e = bbb::launch_bwd_simt(a, (cudaStream_t)stream, sm_count(), &nl);
    if (e != cudaSuccess) return cuda_fail(e, "bwd_simt launch");
    g_launches += nl;
    return BBB_OK;
}

}  // namespace

extern "C" {

size_t bbb_workspace_bytes(const bbb_layer_desc* desc) {
    if (!desc || desc->math == BBB_MATH_FP32) return kBaseWorkspace;
    bbb::Geom g;
    if (!bbb::make_geom(*desc, g)) return kBaseWorkspace;
    const int sets = weight_sets(*desc, g);
    return kTcOffset + (sets > 1 ? sets * set_stride(g) : tc_set_bytes(g));
}

int bbb_conv2d_forward(const bbb_layer_desc* desc, const void* x, const float* W_mu, const float* W_rho,
                       const float* bias_mu, const float* bias_rho, void* y, float* kl_out, float* act_std,
                       const float* eps_a, const float* eps_b, uint64_t seed, uint64_t stream_id, const uint64_t* stream_base,
                       void* workspace, size_t workspace_bytes, void* cuda_stream) {
    return forward_impl(desc, false, x, W_mu, W_rho, bias_mu, bias_rho, y, kl_out, act_std, eps_a, eps_b, seed,
                        stream_id, stream_base, workspace, workspace_bytes, cuda_stream, nullptr);
}

int bbb_linear_forward(const bbb_layer_desc* desc, const void* x, const float* W_mu, const float* W_rho,
                       const float* bias_mu, const float* bias_rho, void* y, float* kl_out, float* act_std,
                       const float* eps_a, const float* eps_b, uint64_t seed, uint64_t stream_id, const uint64_t* stream_base,
                       void* workspace, size_t workspace_bytes, void* cuda_stream) {
    return forward_impl(desc, true, x, W_mu, W_rho, bias_mu, bias_rho, y, kl_out, act_std, eps_a, eps_b, seed,
                        stream_id, stream_base, workspace, workspace_bytes, cuda_stream, nullptr);
}

int bbb_conv2d_forward_prior(const bbb_layer_desc* desc, const void* x, const float* W_mu, const float* W_rho,
                             const float* bias_mu, const float* bias_rho, void* y, float* kl_out, float* act_std,
                             const float* eps_a, const float* eps_b, uint64_t seed, uint64_t stream_id,
                             const uint64_t* stream_base, void* workspace, size_t workspace_bytes, void* cuda_stream,
                             const bbb_prior* prior) {
    return forward_impl(desc, false, x, W_mu, W_rho, bias_mu, bias_rho, y, kl_out, act_std, eps_a, eps_b, seed,
                        stream_id, stream_base, workspace, workspace_bytes, cuda_stream, prior);
}

int bbb_linear_forward_prior(const bbb_layer_desc* desc, const void* x, const float* W_mu, const float* W_rho,
                             const float* bias_mu, const float* bias_rho, void* y, float* kl_out, float* act_std,
                             const float* eps_a, const float* eps_b, uint64_t seed, uint64_t stream_id,
                             const uint64_t* stream_base, void* workspace, size_t workspace_bytes, void* cuda_stream,
                             const bbb_prior* prior) {
    return forward_impl(desc, true, x, W_mu, W_rho, bias_mu, bias_rho, y, kl_out, act_std, eps_a, eps_b, seed,
                        stream_id, stream_base, workspace, workspace_bytes, cuda_stream, prior);
}

int bbb_conv2d_backward(const bbb_layer_desc* desc, const void* x, const void* grad_y, const float* W_mu,
                        const float* W_rho, const float* bias_mu, const float* bias_rho, const float* act_std,
                        const float* eps_a, const float* eps_b, uint64_t seed, uint64_t stream_id, const uint64_t* stream_base, void* grad_x,
                        float* g_W_mu, float* g_W_rho, float* g_bias_mu, float* g_bias_rho, void* workspace,
                        size_t workspace_bytes, void* cuda_stream) {
    return backward_impl(desc, false, x, grad_y, W_mu, W_rho, bias_mu, bias_rho, act_std, eps_a, eps_b, seed,
                         stream_id, stream_base, grad_x, g_W_mu, g_W_rho, g_bias_mu, g_bias_rho, workspace, workspace_bytes,
                         cuda_stream, nullptr);
}

int bbb_linear_backward(const bbb_layer_desc* desc, const void* x, const void* grad_y, const float* W_mu,
                        const float* W_rho, const float* bias_mu, const float* bias_rho, const float* act_std,
                        const float* eps_a, const float* eps_b, uint64_t seed, uint64_t stream_id, const uint64_t* stream_base, void* grad_x,
                        float* g_W_mu, float* g_W_rho, float* g_bias_mu, float* g_bias_rho, void* workspace,
                        size_t workspace_bytes, void* cuda_stream) {
    return backward_impl(desc, true, x, grad_y, W_mu, W_rho, bias_mu, bias_rho, act_std, eps_a, eps_b, seed,
                         stream_id, stream_base, grad_x, g_W_mu, g_W_rho, g_bias_mu, g_bias_rho, workspace, workspace_bytes,
                         cuda_stream, nullptr);
}

int bbb_conv2d_backward_prior(const bbb_layer_desc* desc, const void* x, const void* grad_y, const float* W_mu,
                              const float* W_rho, const float* bias_mu, const float* bias_rho, const float* act_std,
                              const float* eps_a, const float* eps_b, uint64_t seed, uint64_t stream_id,
                              const uint64_t* stream_base, void* grad_x, float* g_W_mu, float* g_W_rho, float* g_bias_mu,
                              float* g_bias_rho, void* workspace, size_t workspace_bytes, void* cuda_stream,
                              const bbb_prior* prior) {
    return backward_impl(desc, false, x, grad_y, W_mu, W_rho, bias_mu, bias_rho, act_std, eps_a, eps_b, seed,
                         stream_id, stream_base, grad_x, g_W_mu, g_W_rho, g_bias_mu, g_bias_rho, workspace, workspace_bytes,
                         cuda_stream, prior);
}
int bbb_linear_backward_prior(const bbb_layer_desc* desc, const void* x, const void* grad_y, const float* W_mu,
                              const float* W_rho, const float* bias_mu, const float* bias_rho, const float* act_std,
                              const float* eps_a, const float* eps_b, uint64_t seed, uint64_t stream_id,
                              const uint64_t* stream_base, void* grad_x, float* g_W_mu, float* g_W_rho, float* g_bias_mu,
                              float* g_bias_rho, void* workspace, size_t workspace_bytes, void* cuda_stream,
                              const bbb_prior* prior) {
    return backward_impl(desc, true, x, grad_y, W_mu, W_rho, bias_mu, bias_rho, act_std, eps_a, eps_b, seed,
                         stream_id, stream_base, grad_x, g_W_mu, g_W_rho, g_bias_mu, g_bias_rho, workspace, workspace_bytes,
                         cuda_stream, prior);
}

/* shape / layout / MC-fold checks of bbb_layer_forward_fused, callable without a GPU (host logic only); `s4` tells
 * whether an NCHW input goes to the stride-4 first-layer kernel rather than the gather path */
static int fused_check(const bbb_layer_desc* d, bbb::Geom& g, int32_t in_layout, int32_t in_pitch, int32_t prev_hw,
                       int32_t out_layout, int32_t out_pitch, bool& s4) {
    s4 = false;
    if (int rc = check_desc(d, g, false)) return rc;
    if (d->math == BBB_MATH_FP32 || d->math == BBB_MATH_TF32_TC) return fail(BBB_E_UNSUPPORTED, "the fused chain exists on the tensor-core (bf16) path only");
    const int pool = d->pool_k != 0;
    if (pool && !(d->pool_k == 2 && d->pool_s == 2)) return fail(BBB_E_UNSUPPORTED, "only a 2x2 stride-2 max-pool can be fused");
    if (pool && ((g.OH | g.OW) & 1)) return fail(BBB_E_UNSUPPORTED, "fused pool needs even output height/width");
    if (out_layout == BBB_LAYOUT_PACKED_BF16 && (g.N % 64 || out_pitch != (pool ? g.OHW / 4 : g.OHW) * g.N))
        return fail(BBB_E_INVALID, "tiled packed output needs Cout %% 64 == 0 and out_pitch == pixels*Cout (got %d)", out_pitch);
    const int out_mode = out_layout == BBB_LAYOUT_PACKED_BF16 ? 0 : (out_layout == BBB_LAYOUT_ROWMAJOR_F32 ? 1 : 2);
    s4 = in_layout == BBB_LAYOUT_NCHW_F32 && s4_enabled() && bbb::conv_s4_supported(*d, g, pool, out_mode == 0);
    if (const int rows = d->reserved[1]; rows > 0) {   // MC samples folded into the batch
        if (!d->sample) return fail(BBB_E_UNSUPPORTED, "MC-sample folding needs a sampling call");
        if (g.B % rows) return fail(BBB_E_INVALID, "batch %d is not a multiple of the rows per MC sample %d", g.B, rows);
        // a row tile (128 rows; 16 images in the stride-4 kernel) must not straddle two weight samples
        if (d->variant == BBB_VARIANT_BBB && rows % 128)
            return fail(BBB_E_UNSUPPORTED, "BBB MC-sample folding needs a multiple of 128 rows per sample (got %d)", rows);
        if (in_layout == BBB_LAYOUT_NCHW_F32 && !s4) return fail(BBB_E_UNSUPPORTED, "MC-sample folding is not available on the gather path");
    }
    if (in_layout == BBB_LAYOUT_NCHW_F32) {
        if (d->act_dtype != BBB_DTYPE_F32) return fail(BBB_E_UNSUPPORTED, "the tensor-core gather path takes fp32 activations only");
        if (!bbb::tc_supported(g)) return fail(BBB_E_UNSUPPORTED, "shape not supported by the tensor-core gather path");
        if (out_mode == 1 && (pool ? g.OHW / 4 : g.OHW) != 1) return fail(BBB_E_UNSUPPORTED, "row-major fp32 output needs a 1x1 map on the gather path");
    } else if (in_layout == BBB_LAYOUT_PACKED_BF16) {
        if (!bbb::fused_supported(g, pool)) return fail(BBB_E_UNSUPPORTED, "shape not supported by the fused tap-GEMM path");
        if (in_pitch != g.HW * g.Cin) return fail(BBB_E_INVALID, "tiled packed input: in_pitch must be pixels*Cin (got %d)", in_pitch);
        if (prev_hw < 1 || g.Cin % prev_hw) return fail(BBB_E_INVALID, "bad prev_hw %d", prev_hw);
    } else {
        return fail(BBB_E_INVALID, "bad in_layout %d", in_layout);
    }
    return BBB_OK;
}

int bbb_forward_supported(const bbb_layer_desc* d) {
    bbb::Geom g;
    int math = BBB_MATH_FP32;
    if (int rc = check_desc(d, g, false)) return rc;
    if (int rc = layer_math(d, g, math)) return rc;
    return layer_fold_check(d, g, math);
}

int bbb_fused_supported(const bbb_layer_desc* d, int32_t in_layout, int32_t in_pitch, int32_t prev_hw,
                        int32_t out_layout, int32_t out_pitch) {
    bbb::Geom g;
    bool s4;
    return fused_check(d, g, in_layout, in_pitch, prev_hw, out_layout, out_pitch, s4);
}

int bbb_layer_forward_fused(const bbb_layer_desc* d, const void* x, const void* x_sq, int32_t in_layout,
                            int32_t in_pitch, int32_t prev_hw, const float* W_mu, const float* W_rho,
                            const float* bias_mu, const float* bias_rho, void* y, void* y_sq, int32_t out_layout,
                            int32_t out_pitch, float* kl_out, const float* eps_a, const float* eps_b, uint64_t seed,
                            uint64_t stream_id, const uint64_t* stream_base, void* ws, size_t ws_bytes, void* stream) {
    return bbb_layer_forward_fused_prior(d, x, x_sq, in_layout, in_pitch, prev_hw, W_mu, W_rho, bias_mu, bias_rho, y, y_sq,
                                         out_layout, out_pitch, kl_out, eps_a, eps_b, seed, stream_id, stream_base, ws,
                                         ws_bytes, stream, nullptr);
}

int bbb_layer_forward_fused_prior(const bbb_layer_desc* d, const void* x, const void* x_sq, int32_t in_layout,
                                  int32_t in_pitch, int32_t prev_hw, const float* W_mu, const float* W_rho,
                                  const float* bias_mu, const float* bias_rho, void* y, void* y_sq, int32_t out_layout,
                                  int32_t out_pitch, float* kl_out, const float* eps_a, const float* eps_b, uint64_t seed,
                                  uint64_t stream_id, const uint64_t* stream_base, void* ws, size_t ws_bytes, void* stream,
                                  const bbb_prior* prior) {
    bbb_layer_desc dcopy;
    Masks mk;
    d = desc_masks(d, prior, dcopy, mk);
    bbb::Geom g;
    bool s4;
    if (int rc = fused_check(d, g, in_layout, in_pitch, prev_hw, out_layout, out_pitch, s4)) return rc;
    const bool prep_only = (d->reserved[0] & BBB_FUSED_PREP_ONLY) != 0, skip_prep = (d->reserved[0] & BBB_FUSED_SKIP_PREP) != 0;
    if (prep_only && skip_prep) return fail(BBB_E_INVALID, "PREP_ONLY and SKIP_PREP are exclusive");
    const bool timed = (d->reserved[0] & BBB_FUSED_NO_TIMELINE) == 0;
    if (!W_mu || !W_rho || (!prep_only && (!x || !y))) return fail(BBB_E_INVALID, "NULL tensor pointer");
    if (d->has_bias && (!bias_mu || !bias_rho)) return fail(BBB_E_INVALID, "has_bias set but bias pointers NULL");
    if (int rc = check_prior(prior, d->has_bias != 0, mk)) return rc;
    const int pool = d->pool_k != 0;
    bbb::McFold fold;                   // rows, samples and path checked by fused_check
    if (int rc = layer_fold(d, g, eps_a, eps_b, fold)) return rc;
    const size_t need = bbb_workspace_bytes(d);
    if (!ws || ws_bytes < need) return fail(BBB_E_WORKSPACE, "workspace too small for the fused path: need %zu bytes", need);
    if (out_layout == BBB_LAYOUT_PACKED_BF16 && y_sq && y_sq != (void*)((__nv_bfloat16*)y + 128 * 64))
        return fail(BBB_E_INVALID, "tiled packed output with squares: the planes are interleaved, y_sq must be y + 8192 elements");
    cudaStream_t st = (cudaStream_t)stream;
    const int out_mode = out_layout == BBB_LAYOUT_PACKED_BF16 ? 0 : (out_layout == BBB_LAYOUT_ROWMAJOR_F32 ? 1 : 2);
    int nl = 0;
    if (s4) {
        // stride-4 first layer: the tensor core reads its A operand straight from the staged image (conv_s4_tc.cuh)
        bbb::S4Args a;
        layer_args(a, d, g, W_mu, W_rho, bias_mu, bias_rho, kl_out, eps_a, eps_b, seed, stream_id, stream_base, ws,
                   bbb::conv_s4_bias_offset(g), fold, "conv_s4_prep", timed && !skip_prep, "conv_s4", timed && !prep_only);
        a.x = (const float*)x; a.y = y; a.y_sq = y_sq; a.out_pitch = out_pitch;
        cudaError_t e = bbb::launch_conv_s4(a, st, !skip_prep, !prep_only, &nl, prior_ptrs(prior, kl_out, mk));
        if (e != cudaSuccess) return cuda_fail(e, "conv_s4 launch");
    } else if (in_layout == BBB_LAYOUT_NCHW_F32) {
        bbb::TcArgs a;                  // fold.rows = 0: fused_check refuses a fold on the gather path
        layer_args(a, d, g, W_mu, W_rho, bias_mu, bias_rho, kl_out, eps_a, eps_b, seed, stream_id, stream_base, ws,
                   bbb::tc_bias_offset(g, false), fold, "weight_prep", timed && !skip_prep, "gemm_tc", timed && !prep_only);
        a.x = x; a.y = y; a.act_std = nullptr; a.act_dtype = d->act_dtype; a.tf32 = 0;
        a.skip_prep = skip_prep; a.prep_only = prep_only; a.y_sq = y_sq; a.out_mode = out_mode == 1 ? 2 : out_mode; a.out_pitch = out_pitch; a.pool = pool;
        cudaError_t e = bbb::launch_fwd_tc(a, st, sm_count(), &nl, prior_ptrs(prior, kl_out, mk));
        if (e != cudaSuccess) return cuda_fail(e, "fused gather launch");
    } else if (in_layout == BBB_LAYOUT_PACKED_BF16) {
        bbb::FusedArgs a;
        layer_args(a, d, g, W_mu, W_rho, bias_mu, bias_rho, kl_out, eps_a, eps_b, seed, stream_id, stream_base, ws,
                   bbb::fused_bias_offset(g), fold, "tap_prep", timed && !skip_prep, "tap_gemm", timed && !prep_only);
        a.prev_hw = prev_hw; a.y = y; a.y_sq = y_sq; a.out_mode = out_mode; a.out_pitch = out_pitch; a.pool = pool;
        a.in_pitch = in_pitch;
        const char* why = "";
        cudaError_t e = bbb::launch_fused(a, x, x_sq, st, &nl, &why, !skip_prep, !prep_only, sm_count(), g_wide_tiles.load() != 0,
                                          prior_ptrs(prior, kl_out, mk));
        if (e != cudaSuccess) return fail(BBB_E_CUDA, "fused tap-GEMM launch: %s %s", cudaGetErrorString(e), why);
    } else {
        return fail(BBB_E_INVALID, "bad in_layout %d", in_layout);
    }
    g_launches += nl;
    return BBB_OK;
}

int bbb_kl_forward(const float* W_mu, const float* W_rho, uint64_t n_w, const float* bias_mu,
                   const float* bias_rho, uint64_t n_b, float prior_mu, float prior_sigma, int32_t kl_convention,
                   float* kl_out, void* workspace, size_t workspace_bytes, void* cuda_stream) {
    return bbb_kl_forward_prior(W_mu, W_rho, n_w, bias_mu, bias_rho, n_b, prior_mu, prior_sigma, kl_convention, kl_out,
                                workspace, workspace_bytes, cuda_stream, nullptr);
}

int bbb_kl_forward_prior(const float* W_mu, const float* W_rho, uint64_t n_w, const float* bias_mu,
                         const float* bias_rho, uint64_t n_b, float prior_mu, float prior_sigma, int32_t kl_convention,
                         float* kl_out, void* workspace, size_t workspace_bytes, void* cuda_stream, const bbb_prior* prior) {
    const Masks mk = take_masks(prior, kl_convention);
    if (!W_mu || !W_rho || !kl_out) return fail(BBB_E_INVALID, "NULL tensor pointer");
    if (n_b && (!bias_mu || !bias_rho)) return fail(BBB_E_INVALID, "n_b > 0 but bias pointers NULL");
    if (int rc = check_prior(prior, n_b > 0, mk)) return rc;
    if (!workspace || workspace_bytes < kBaseWorkspace) return fail(BBB_E_WORKSPACE, "workspace too small: need %zu bytes", kBaseWorkspace);
    const bool tensor_prior = prior && prior->w_mu, masked = mk.w != nullptr;
    if (!tensor_prior && !(prior_sigma > 0.0f)) return fail(BBB_E_INVALID, "prior_sigma must be > 0");
    const uint64_t work = (n_w + 3) / 4 + n_b;
    uint64_t blocks = (work + 255) / 256;
    const uint64_t cap = (uint64_t)sm_count() * 8;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    if (blocks > kMaxKlSlots) blocks = kMaxKlSlots;
    double* partials = (double*)((char*)workspace + kCounterBytes);
    if (masked && tensor_prior)
        bbb::kl_forward_masked_kernel<true><<<(unsigned)blocks, 256, 0, (cudaStream_t)cuda_stream>>>(
            W_mu, W_rho, n_w, bias_mu, bias_rho, n_b, 0.0f, 1.0f, prior_ptrs(prior, kl_out, mk), kl_convention, partials,
            (unsigned int*)workspace, kl_out);
    else if (masked)
        bbb::kl_forward_masked_kernel<false><<<(unsigned)blocks, 256, 0, (cudaStream_t)cuda_stream>>>(
            W_mu, W_rho, n_w, bias_mu, bias_rho, n_b, prior_mu, prior_sigma, prior_ptrs(prior, kl_out, mk), kl_convention,
            partials, (unsigned int*)workspace, kl_out);
    else if (prior)
        bbb::kl_forward_prior_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)cuda_stream>>>(
            W_mu, W_rho, n_w, bias_mu, bias_rho, n_b, prior_ptrs(prior, kl_out), kl_convention, partials,
            (unsigned int*)workspace, kl_out);
    else
        bbb::kl_forward_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)cuda_stream>>>(
            W_mu, W_rho, n_w, bias_mu, bias_rho, n_b, prior_mu, prior_sigma, kl_convention, partials,
            (unsigned int*)workspace, kl_out);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return cuda_fail(e, "kl_forward launch");
    g_launches += 1;
    return BBB_OK;
}

int bbb_kl_backward(const float* mu, const float* rho, uint64_t n, float prior_mu, float prior_sigma,
                    int32_t kl_convention, const float* grad_kl, float* g_mu, float* g_rho, void* cuda_stream) {
    return bbb_kl_backward_prior(mu, rho, n, prior_mu, prior_sigma, kl_convention, grad_kl, g_mu, g_rho, cuda_stream,
                                 nullptr);
}

int bbb_kl_backward_prior(const float* mu, const float* rho, uint64_t n, float prior_mu, float prior_sigma,
                          int32_t kl_convention, const float* grad_kl, float* g_mu, float* g_rho, void* cuda_stream,
                          const bbb_prior* prior) {
    const Masks mk = take_masks(prior, kl_convention);
    if (!mu || !rho || !grad_kl || !g_mu || !g_rho) return fail(BBB_E_INVALID, "NULL tensor pointer");
    if (int rc = check_prior(prior, false, mk)) return rc;   // the n elements' prior is prior->w_mu / w_sigma
    if (n == 0) return BBB_OK;
    uint64_t blocks = (n + 255) / 256;
    const uint64_t cap = (uint64_t)sm_count() * 8;
    if (blocks > cap) blocks = cap;
    const bool tensor_prior = prior && prior->w_mu;
    if (mk.w)
        (tensor_prior ? bbb::kl_backward_masked_kernel<true> : bbb::kl_backward_masked_kernel<false>)
            <<<(unsigned)blocks, 256, 0, (cudaStream_t)cuda_stream>>>(mu, rho, n, prior_mu, prior_sigma, prior->w_mu,
                                                                      prior->w_sigma, mk.w, kl_convention,
                                                                      grad_kl, g_mu, g_rho);
    else if (prior)
        bbb::kl_backward_prior_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)cuda_stream>>>(
            mu, rho, n, prior->w_mu, prior->w_sigma, kl_convention, grad_kl, g_mu, g_rho);
    else
        bbb::kl_backward_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)cuda_stream>>>(
            mu, rho, n, prior_mu, prior_sigma, kl_convention, grad_kl, g_mu, g_rho);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return cuda_fail(e, "kl_backward launch");
    g_launches += 1;
    return BBB_OK;
}

size_t bbb_kl_mc_workspace_bytes(int32_t n_draws) {
    const size_t d = n_draws > 0 ? (size_t)n_draws : 1;
    return kl_mc_counter_bytes(d) + d * kMaxKlSlots * sizeof(double);
}

int bbb_kl_mc_forward(const float* W_mu, const float* W_rho, uint64_t n_w, const float* bias_mu, const float* bias_rho,
                      uint64_t n_b, const bbb_mixture_prior* prior, uint64_t seed, uint64_t stream_id,
                      const uint64_t* stream_base, int32_t n_draws, uint64_t draw_stride, float* kl_out, void* workspace,
                      size_t workspace_bytes, void* cuda_stream) {
    if (!W_mu || !W_rho || !kl_out) return fail(BBB_E_INVALID, "NULL tensor pointer");
    if (n_b && (!bias_mu || !bias_rho)) return fail(BBB_E_INVALID, "n_b > 0 but bias pointers NULL");
    bbb::MixPrior q;
    if (int rc = check_mixture(prior, n_draws, q)) return rc;
    const size_t need = bbb_kl_mc_workspace_bytes(n_draws);
    if (!workspace || workspace_bytes < need) return fail(BBB_E_WORKSPACE, "workspace too small: need %zu bytes", need);
    const uint64_t work = n_w / 4 + n_w % 4 + n_b;
    uint64_t blocks = (work + bbb::KL_MC_THREADS - 1) / bbb::KL_MC_THREADS;
    const uint64_t cap = (uint64_t)sm_count() * 8;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    if (blocks > kMaxKlSlots) blocks = kMaxKlSlots;
    unsigned int* counters = (unsigned int*)workspace;
    double* partials = (double*)((char*)workspace + kl_mc_counter_bytes((size_t)n_draws));
    // the draws go in launches of at most KL_MC_MAX_DRAWS, each draw with its own counter and partial row
    for (int32_t d0 = 0; d0 < n_draws; d0 += bbb::KL_MC_MAX_DRAWS) {
        const int nd = std::min<int32_t>(bbb::KL_MC_MAX_DRAWS, n_draws - d0);
        bbb::kl_mc_forward_kernel<<<(unsigned)blocks, bbb::KL_MC_THREADS, (size_t)nd * bbb::KL_MC_THREADS * sizeof(double),
                                    (cudaStream_t)cuda_stream>>>(
            W_mu, W_rho, n_w, bias_mu, bias_rho, n_b, q, bbb::make_key(seed, stream_id + (uint64_t)d0 * draw_stride),
            (const unsigned long long*)stream_base, nd, draw_stride, counters + d0, partials + (size_t)d0 * kMaxKlSlots,
            kl_out + d0);
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return cuda_fail(e, "kl_mc_forward launch");
        g_launches += 1;
    }
    return BBB_OK;
}

int bbb_kl_mc_backward(const float* mu, const float* rho, uint64_t n, uint64_t first_element,
                       const bbb_mixture_prior* prior, uint64_t seed, uint64_t stream_id, const uint64_t* stream_base,
                       int32_t n_draws, uint64_t draw_stride, const float* grad_kl, float* g_mu, float* g_rho,
                       void* cuda_stream) {
    if (!mu || !rho || !grad_kl || !g_mu || !g_rho) return fail(BBB_E_INVALID, "NULL tensor pointer");
    bbb::MixPrior q;
    if (int rc = check_mixture(prior, n_draws, q)) return rc;
    if (n == 0) return BBB_OK;
    uint64_t blocks = ((n + 3) / 4 + bbb::KL_MC_THREADS - 1) / bbb::KL_MC_THREADS;
    const uint64_t cap = (uint64_t)sm_count() * 8;
    if (blocks > cap) blocks = cap;
    bbb::kl_mc_backward_kernel<<<(unsigned)blocks, bbb::KL_MC_THREADS, 0, (cudaStream_t)cuda_stream>>>(
        mu, rho, n, first_element, q, bbb::make_key(seed, stream_id), (const unsigned long long*)stream_base, n_draws,
        draw_stride, grad_kl, g_mu, g_rho);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return cuda_fail(e, "kl_mc_backward launch");
    g_launches += 1;
    return BBB_OK;
}

int bbb_philox_normal_fill(float* out, uint64_t n, uint64_t seed, uint64_t stream_id, uint64_t offset,
                           void* cuda_stream) {
    if (!out) return fail(BBB_E_INVALID, "NULL output pointer");
    if (n == 0) return BBB_OK;
    uint64_t blocks = (n + 255) / 256;
    const uint64_t cap = (uint64_t)sm_count() * 8;
    if (blocks > cap) blocks = cap;
    bbb::philox_fill_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)cuda_stream>>>(out, n, bbb::make_key(seed, stream_id), offset);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return cuda_fail(e, "philox_fill launch");
    g_launches += 1;
    return BBB_OK;
}

int bbb_lrt_noise_grad(const bbb_layer_desc* d, const float* grad_y, const float* act_std, uint64_t seed,
                       uint64_t stream_id, const uint64_t* stream_base, float* gv, void* cuda_stream) {
    bbb::Geom g;
    if (int rc = check_desc(d, g, false)) return rc;        // first image and fold within int32 element counts
    if (d->variant != BBB_VARIANT_LRT) return fail(BBB_E_INVALID, "bbb_lrt_noise_grad: not an LRT layer desc (variant %d)", d->variant);
    if (!d->sample) return fail(BBB_E_UNSUPPORTED, "bbb_lrt_noise_grad: a mean-only call (sample == 0) draws no noise");
    const int rows = d->reserved[1];
    if (rows > 0 && g.B % rows) return fail(BBB_E_INVALID, "batch %d is not a multiple of the rows per MC sample %d", g.B, rows);
    if (!grad_y || !act_std || !gv) return fail(BBB_E_INVALID, "NULL tensor pointer");
    bbb::McFold fold;
    if (int rc = layer_fold(d, g, nullptr, nullptr, fold)) return rc;
    const bool vec4 = g.N % 4 == 0;
    const uint64_t work = (uint64_t)g.B * (vec4 ? g.N / 4 : g.N) * g.OHW;
    uint64_t blocks = (work + 255) / 256;
    const uint64_t cap = (uint64_t)sm_count() * 8;
    if (blocks > cap) blocks = cap;
    const bbb::NoiseKey key = bbb::make_key(seed, stream_id);
    const auto* base = (const unsigned long long*)stream_base;
    if (vec4)
        bbb::lrt_noise_grad_kernel<true><<<(unsigned)blocks, 256, 0, (cudaStream_t)cuda_stream>>>(
            grad_y, act_std, gv, g.B, g.N, g.OHW, key, base, fold);
    else
        bbb::lrt_noise_grad_kernel<false><<<(unsigned)blocks, 256, 0, (cudaStream_t)cuda_stream>>>(
            grad_y, act_std, gv, g.B, g.N, g.OHW, key, base, fold);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return cuda_fail(e, "lrt_noise_grad launch");
    g_launches += 1;
    return BBB_OK;
}

int bbb_mc_combine(const float* logits, int32_t S, int32_t B, int32_t C, float* log_outputs, float* moments,
                   void* cuda_stream) {
    if (!logits || !log_outputs) return fail(BBB_E_INVALID, "NULL tensor pointer");
    if (S <= 0 || B <= 0 || C <= 0) return fail(BBB_E_INVALID, "bad S/B/C");
    if ((size_t)S * sizeof(float) > 40000) return fail(BBB_E_UNSUPPORTED, "S too large");
    bbb::mc_combine_kernel<<<B, 128, S * sizeof(float), (cudaStream_t)cuda_stream>>>(logits, S, B, C, log_outputs, moments);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return cuda_fail(e, "mc_combine launch");
    g_launches += 1;
    return BBB_OK;
}

size_t bbb_mc_buffer_bytes(int32_t B, int32_t C, int32_t flags, int32_t world) {
    if (B <= 0 || C <= 0 || world <= 0 || world > bbb::MCX_MAX_RANKS) return 0;
    if ((flags & BBB_MC_INFO) && !(flags & BBB_MC_MOMENTS)) return 0;
    return bbb::mcx_buffer_bytes(B, C, flags & BBB_MC_MOMENTS, world, (flags & BBB_MC_INFO) != 0);
}
size_t bbb_mc_state_bytes(void) { return 64 + (size_t)bbb::MCX_MAX_CTAS * 2 * sizeof(double); }

// bbb_mc_exchange_info and bbb_mc_exchange_sharded: batch_shards == 1 launches the default kernels
static int mc_exchange_impl(const float* logits, int32_t S_local, int32_t S_total, int32_t B, int32_t C, const float* kl,
                            int32_t n_kl, int32_t flags, const int64_t* labels, float train_size, float beta, int32_t rank,
                            int32_t world, void* const* peer_buffers, void* state, float* log_outputs, float* kl_out,
                            float* pred, float* epistemic, float* aleatoric, float* entropy, float* head,
                            uint64_t* noise_base, uint64_t noise_inc, float* expected_entropy, float* mutual_info,
                            int32_t batch_shards, double* metrics, void* cuda_stream) {
    if (!log_outputs || !peer_buffers || !state) return fail(BBB_E_INVALID, "NULL pointer");
    if (batch_shards < 1 || world % batch_shards) return fail(BBB_E_INVALID, "world %d is not a multiple of batch_shards %d", world, batch_shards);
    if (batch_shards > B) return fail(BBB_E_INVALID, "batch_shards %d > B %d: a row block would be empty", batch_shards, B);
    if (S_local < 0 || S_total <= 0 || B <= 0 || C <= 0) return fail(BBB_E_INVALID, "bad S/B/C");
    if (S_local > 0 && !logits) return fail(BBB_E_INVALID, "S_local > 0 but logits is NULL");
    if (S_local > bbb::MCX_MAX_SLOCAL) return fail(BBB_E_UNSUPPORTED, "more than %d local samples per call", bbb::MCX_MAX_SLOCAL);
    if (world < 1 || world > bbb::MCX_MAX_RANKS || rank < 0 || rank >= world) return fail(BBB_E_INVALID, "bad rank/world %d/%d", rank, world);
    if ((pred || epistemic || aleatoric || entropy) && !(flags & BBB_MC_MOMENTS))
        return fail(BBB_E_INVALID, "uncertainty outputs need BBB_MC_MOMENTS");
    const bool info = (flags & BBB_MC_INFO) != 0;
    if (info && !(flags & BBB_MC_MOMENTS)) return fail(BBB_E_INVALID, "BBB_MC_INFO needs BBB_MC_MOMENTS");
    if ((expected_entropy || mutual_info) && !info)
        return fail(BBB_E_INVALID, "expected_entropy / mutual_info need BBB_MC_INFO");
    bbb::McxArgs a;
    a.logits = logits; a.kl = kl; a.n_kl = kl ? (n_kl > 0 ? n_kl : 1) : 0; a.S_local = S_local; a.S_total = S_total; a.B = B; a.C = C;
    a.want_moments = (flags & BBB_MC_MOMENTS) ? 1 : 0; a.normalized = (flags & BBB_MC_NORMALIZED) ? 1 : 0;
    a.labels = (const long long*)labels; a.train_size = train_size; a.beta = beta; a.rank = rank; a.world = world;
    for (int q = 0; q < bbb::MCX_MAX_RANKS; ++q) a.peer[q] = q < world ? (unsigned char*)peer_buffers[q] : nullptr;
    for (int q = 0; q < world; ++q) if (!a.peer[q]) return fail(BBB_E_INVALID, "peer buffer %d is NULL", q);
    a.seq = (unsigned int*)state; a.done = (unsigned int*)state + 1; a.timeouts = (unsigned int*)state + 2;
    a.noise_base = nullptr; a.noise_inc = 0;
    if (noise_base) { a.noise_base = (unsigned long long*)noise_base; a.noise_inc = noise_inc; }
    a.timeout_ns = 10ull * 1000 * 1000 * 1000;
    if (const char* e = getenv("BBB_B200_MC_TIMEOUT_MS")) a.timeout_ns = (unsigned long long)atoll(e) * 1000000ull;
    a.head_partials = (double*)((char*)state + 64);
    a.log_outputs = log_outputs; a.kl_out = kl_out; a.pred = pred; a.epistemic = epistemic; a.aleatoric = aleatoric;
    a.entropy = entropy; a.head = head; a.trace = g_mcx_trace;
    a.expected_entropy = expected_entropy; a.mutual_info = mutual_info; a.metrics = metrics;
    // row blocks: rank r = sample group r % Rs, row block r / Rs; blocks as equal as possible, the first B % Rb one longer
    const int Rs = world / batch_shards, blk = rank / Rs, per = B / batch_shards, rem = B % batch_shards;
    a.groups = Rs; a.group = rank % Rs; a.block = blk;
    a.row0 = blk * per + (blk < rem ? blk : rem); a.rows = per + (blk < rem ? 1 : 0);
    { bbb::Geom tg = {}; tg.M = B; tg.N = C; tg.K = S_local; a.tl = tl_slot(true, "mc_exchange", tg); }
    // the grid depends on B only: CTA c of every rank finishes the same images.  At most MCX_MAX_CTAS CTAs: all
    // co-resident, so a CTA spinning on a peer's word never keeps that peer's producer off an SM.
    int grid = (B + bbb::MCX_THREADS / 32 - 1) / (bbb::MCX_THREADS / 32);
    if (grid > bbb::MCX_MAX_CTAS) grid = bbb::MCX_MAX_CTAS;
    const bool shard = batch_shards > 1;
    auto kern = metrics ? (shard ? (info ? bbb::mc_exchange_kernel<true, true, true> : bbb::mc_exchange_kernel<false, true, true>)
                                 : (info ? bbb::mc_exchange_kernel<true, false, true> : bbb::mc_exchange_kernel<false, false, true>))
                        : shard ? (info ? bbb::mc_exchange_kernel<true, true> : bbb::mc_exchange_kernel<false, true>)
                                : (info ? bbb::mc_exchange_kernel<true> : bbb::mc_exchange_kernel<false>);
    cudaError_t e = bbb::launch_pdl(kern,
                                     dim3(grid), dim3(bbb::MCX_THREADS), bbb::mcx_smem_bytes(S_local, metrics != nullptr),
                                     (cudaStream_t)cuda_stream, a);
    if (e == cudaSuccess) e = cudaGetLastError();
    if (e != cudaSuccess) return cuda_fail(e, "mc_exchange launch");
    g_launches += 1;
    return BBB_OK;
}
int bbb_mc_exchange_info(const float* logits, int32_t S_local, int32_t S_total, int32_t B, int32_t C, const float* kl,
                         int32_t n_kl, int32_t flags, const int64_t* labels, float train_size, float beta, int32_t rank,
                         int32_t world, void* const* peer_buffers, void* state, float* log_outputs, float* kl_out, float* pred,
                         float* epistemic, float* aleatoric, float* entropy, float* head, uint64_t* noise_base,
                         uint64_t noise_inc, float* expected_entropy, float* mutual_info, void* cuda_stream) {
    return mc_exchange_impl(logits, S_local, S_total, B, C, kl, n_kl, flags, labels, train_size, beta, rank, world,
                            peer_buffers, state, log_outputs, kl_out, pred, epistemic, aleatoric, entropy, head, noise_base,
                            noise_inc, expected_entropy, mutual_info, 1, nullptr, cuda_stream);
}
int bbb_mc_exchange_sharded(const float* logits, int32_t S_local, int32_t S_total, int32_t B, int32_t C, const float* kl,
                            int32_t n_kl, int32_t flags, const int64_t* labels, float train_size, float beta, int32_t rank,
                            int32_t world, void* const* peer_buffers, void* state, float* log_outputs, float* kl_out,
                            float* pred, float* epistemic, float* aleatoric, float* entropy, float* head,
                            uint64_t* noise_base, uint64_t noise_inc, float* expected_entropy, float* mutual_info,
                            int32_t batch_shards, void* cuda_stream) {
    return mc_exchange_impl(logits, S_local, S_total, B, C, kl, n_kl, flags, labels, train_size, beta, rank, world,
                            peer_buffers, state, log_outputs, kl_out, pred, epistemic, aleatoric, entropy, head, noise_base,
                            noise_inc, expected_entropy, mutual_info, batch_shards, nullptr, cuda_stream);
}
static_assert(BBB_MC_CAL_BINS == bbb::MCM_BINS, "calibration bins: header and kernel disagree");
size_t bbb_mc_metrics_bytes(void) { return bbb::mcm_bytes(); }
int bbb_mc_exchange_metrics(const float* logits, int32_t S_local, int32_t S_total, int32_t B, int32_t C, const float* kl,
                            int32_t n_kl, int32_t flags, const int64_t* labels, float train_size, float beta, int32_t rank,
                            int32_t world, void* const* peer_buffers, void* state, float* log_outputs, float* kl_out,
                            float* pred, float* epistemic, float* aleatoric, float* entropy, float* head,
                            uint64_t* noise_base, uint64_t noise_inc, float* expected_entropy, float* mutual_info,
                            int32_t batch_shards, double* metrics, void* cuda_stream) {
    if (!metrics) return fail(BBB_E_INVALID, "metrics is NULL");
    if (!labels) return fail(BBB_E_INVALID, "metrics need labels");
    return mc_exchange_impl(logits, S_local, S_total, B, C, kl, n_kl, flags, labels, train_size, beta, rank, world,
                            peer_buffers, state, log_outputs, kl_out, pred, epistemic, aleatoric, entropy, head, noise_base,
                            noise_inc, expected_entropy, mutual_info, batch_shards, metrics, cuda_stream);
}
int bbb_mc_exchange(const float* logits, int32_t S_local, int32_t S_total, int32_t B, int32_t C, const float* kl,
                    int32_t n_kl, int32_t flags, const int64_t* labels, float train_size, float beta, int32_t rank, int32_t world,
                    void* const* peer_buffers, void* state, float* log_outputs, float* kl_out, float* pred,
                    float* epistemic, float* aleatoric, float* entropy, float* head, uint64_t* noise_base,
                    uint64_t noise_inc, void* cuda_stream) {
    return bbb_mc_exchange_info(logits, S_local, S_total, B, C, kl, n_kl, flags, labels, train_size, beta, rank, world,
                                peer_buffers, state, log_outputs, kl_out, pred, epistemic, aleatoric, entropy, head,
                                noise_base, noise_inc, nullptr, nullptr, cuda_stream);
}

int bbb_comm_alloc(size_t bytes, void** dev_ptr) {
    if (!dev_ptr || bytes == 0) return fail(BBB_E_INVALID, "bad arguments");
    cudaError_t e = cudaMalloc(dev_ptr, bytes);
    if (e != cudaSuccess) return cuda_fail(e, "cudaMalloc");
    e = cudaMemset(*dev_ptr, 0, bytes);
    if (e != cudaSuccess) return cuda_fail(e, "cudaMemset");
    e = cudaDeviceSynchronize();
    if (e != cudaSuccess) return cuda_fail(e, "cudaDeviceSynchronize");
    return BBB_OK;
}
int bbb_comm_free(void* dev_ptr) {
    cudaError_t e = cudaFree(dev_ptr);
    return e == cudaSuccess ? BBB_OK : cuda_fail(e, "cudaFree");
}
int bbb_comm_export(void* dev_ptr, void* handle64_host) {
    if (!dev_ptr || !handle64_host) return fail(BBB_E_INVALID, "NULL pointer");
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
    cudaIpcMemHandle_t h;
    cudaError_t e = cudaIpcGetMemHandle(&h, dev_ptr);
    if (e != cudaSuccess) return cuda_fail(e, "cudaIpcGetMemHandle");
    memcpy(handle64_host, &h, 64);
    return BBB_OK;
}
int bbb_comm_import(const void* handle64_host, void** peer_ptr) {
    if (!handle64_host || !peer_ptr) return fail(BBB_E_INVALID, "NULL pointer");
    cudaIpcMemHandle_t h;
    memcpy(&h, handle64_host, 64);
    cudaError_t e = cudaIpcOpenMemHandle(peer_ptr, h, cudaIpcMemLazyEnablePeerAccess);
    return e == cudaSuccess ? BBB_OK : cuda_fail(e, "cudaIpcOpenMemHandle");
}
int bbb_comm_unimport(void* peer_ptr) {
    cudaError_t e = cudaIpcCloseMemHandle(peer_ptr);
    return e == cudaSuccess ? BBB_OK : cuda_fail(e, "cudaIpcCloseMemHandle");
}

int bbb_noise_advance(uint64_t* base, uint64_t inc, void* cuda_stream) {
    if (!base) return fail(BBB_E_INVALID, "NULL base pointer");
    bbb::noise_advance_kernel<<<1, 1, 0, (cudaStream_t)cuda_stream>>>((unsigned long long*)base, (unsigned long long)inc);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return cuda_fail(e, "noise_advance launch");
    g_launches += 1;
    return BBB_OK;
}

int bbb_mc_graph_step(void* caller_stream, void* run_stream, void* in_ready, void* wait_a, void* wait_b,
                      void* chain_exec, void* chain_done, void* result_stream, void* exch_exec, void* exch_done) {
    if (!chain_exec || !chain_done || !exch_exec || !exch_done || (run_stream != caller_stream && !in_ready))
        return fail(BBB_E_INVALID, "bbb_mc_graph_step: NULL graph or event");
    const cudaStream_t cur = (cudaStream_t)caller_stream, run = (cudaStream_t)run_stream, rs = (cudaStream_t)result_stream;
    cudaError_t e = cudaSuccess;
    if (run != cur) {
        e = cudaEventRecord((cudaEvent_t)in_ready, cur);
        if (e == cudaSuccess) e = cudaStreamWaitEvent(run, (cudaEvent_t)in_ready, 0);
    }
    if (e == cudaSuccess && wait_a) e = cudaStreamWaitEvent(run, (cudaEvent_t)wait_a, 0);
    if (e == cudaSuccess && wait_b) e = cudaStreamWaitEvent(run, (cudaEvent_t)wait_b, 0);
    if (e == cudaSuccess) e = cudaGraphLaunch((cudaGraphExec_t)chain_exec, run);
    if (e == cudaSuccess) e = cudaEventRecord((cudaEvent_t)chain_done, run);
    if (e == cudaSuccess) e = cudaStreamWaitEvent(rs, (cudaEvent_t)chain_done, 0);
    if (e == cudaSuccess) e = cudaGraphLaunch((cudaGraphExec_t)exch_exec, rs);
    if (e == cudaSuccess) e = cudaEventRecord((cudaEvent_t)exch_done, rs);
    return e == cudaSuccess ? BBB_OK : cuda_fail(e, "bbb_mc_graph_step");
}

/* debug only (not in the public header): per-CTA clock64 checkpoints of tap_gemm_kernel */
void bbb_debug_set_trace(void* dev_ptr) { g_trace = (long long*)dev_ptr; }
void bbb_debug_set_mcx_trace(void* dev_ptr) { g_mcx_trace = (long long*)dev_ptr; }
/* debug only: timeline slots (4 x int64 per instrumented launch; caller presets [INT64_MAX, 0, INT64_MAX, 0] before a run) */
void bbb_debug_set_timeline(void* dev_ptr, int capacity) { g_tl = (long long*)dev_ptr; g_tl_cap = capacity; g_tl_n = 0; }
int bbb_debug_timeline_count(void) { return g_tl_n; }
const char* bbb_debug_timeline_name(int k) { return (k >= 0 && k < g_tl_n) ? g_tl_names[k] : ""; }

const char* bbb_last_error(void) { return g_err; }
int32_t bbb_abi_version(void) { return BBB_ABI_VERSION; }
uint64_t bbb_launch_count(void) { return g_launches.load(); }
int32_t bbb_set_wide_tiles(int32_t prefer_wide) { return g_wide_tiles.exchange(prefer_wide ? 1 : 0); }

}  // extern "C"
