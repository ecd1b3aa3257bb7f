// Shared device helpers: geometry, Philox4x32-10 noise, softplus, KL terms.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <type_traits>
#include "../../include/bbb_b200.h"

namespace bbb {

// Implicit-GEMM view of one layer call: M = batch*OH*OW rows (output pixels),
// N = Cout, K = Cin*KH*KW with k = (c*KH + r)*KW + s -- the OIHW flattening, so
// the weight matrix is [N, K] row-major exactly as stored by the reference.
struct Geom {
    int B, Cin, H, W, Cout, KH, KW, SH, SW, PH, PW, DH, DW, OH, OW;
    int M, N, K, KHW, OHW, HW;
    int linear_like;   // KH=KW=H=W=1, no padding: A[m,k] = x[m*K + k]
};

__host__ inline bool make_geom(const bbb_layer_desc& d, Geom& g) {
    g.B = d.batch; g.Cin = d.in_channels; g.H = d.in_h; g.W = d.in_w; g.Cout = d.out_channels;
    g.KH = d.kernel_h; g.KW = d.kernel_w; g.SH = d.stride_h; g.SW = d.stride_w;
    g.PH = d.pad_h; g.PW = d.pad_w; g.DH = d.dil_h; g.DW = d.dil_w;
    if (g.B <= 0 || g.Cin <= 0 || g.H <= 0 || g.W <= 0 || g.Cout <= 0 || g.KH <= 0 || g.KW <= 0 ||
        g.SH <= 0 || g.SW <= 0 || g.PH < 0 || g.PW < 0 || g.DH <= 0 || g.DW <= 0) return false;
    long oh = ((long)g.H + 2L * g.PH - (long)g.DH * (g.KH - 1) - 1) / g.SH + 1;
    long ow = ((long)g.W + 2L * g.PW - (long)g.DW * (g.KW - 1) - 1) / g.SW + 1;
    if (oh <= 0 || ow <= 0) return false;
    g.OH = (int)oh; g.OW = (int)ow;
    g.OHW = g.OH * g.OW; g.HW = g.H * g.W; g.KHW = g.KH * g.KW;
    long M = (long)g.B * g.OHW, K = (long)g.Cin * g.KHW;
    if (M > 0x7fffffffL || K > 0x7fffffffL || (long)g.B * g.Cin * g.HW > 0x7fffffffL ||
        M * g.Cout > 0x7fffffffL) return false;
    g.M = (int)M; g.N = g.Cout; g.K = (int)K;
    g.linear_like = (g.KH == 1 && g.KW == 1 && g.H == 1 && g.W == 1 && g.PH == 0 && g.PW == 0);
    return true;
}

// ---------------------------------------------------------------- Philox ----
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
    for (int i = 0; i < 10; ++i) {
        const uint32_t hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
        const uint32_t hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
        c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
        k.x += 0x9E3779B9u; k.y += 0xBB67AE85u;
    }
    return c;
}

__device__ __forceinline__ void box_muller(uint32_t a, uint32_t b, float& z0, float& z1) {
    const float u1 = __fmaf_rn((float)(a >> 8), 5.9604644775390625e-08f, 2.98023223876953125e-08f);
    const float u2 = __fmaf_rn((float)(b >> 8), 5.9604644775390625e-08f, 2.98023223876953125e-08f);
    const float rad = sqrtf(__fmul_rn(-2.0f, __logf(u1)));
    float s, c;
    __sincosf(__fmul_rn(6.283185307179586f, u2), &s, &c);
    z0 = __fmul_rn(rad, c);
    z1 = __fmul_rn(rad, s);
}

struct NoiseKey { uint32_t seed_lo, seed_hi, stream_lo, stream_hi; };
__host__ __device__ inline NoiseKey make_key(uint64_t seed, uint64_t stream) {
    NoiseKey k; k.seed_lo = (uint32_t)seed; k.seed_hi = (uint32_t)(seed >> 32);
    k.stream_lo = (uint32_t)stream; k.stream_hi = (uint32_t)(stream >> 32); return k;
}

// graph-replay support: effective stream = stream + *base (base nullable, device memory)
__device__ __forceinline__ NoiseKey effective_key(NoiseKey k, const unsigned long long* base) {
    if (base) {
        const unsigned long long s = (((unsigned long long)k.stream_hi << 32) | k.stream_lo) + __ldg(base);
        k.stream_lo = (uint32_t)s; k.stream_hi = (uint32_t)(s >> 32);
    }
    return k;
}

// Monte-Carlo samples folded into the batch (S samples of a batch are one launch over S*rows rows): row b of the folded
// batch is image b % rows of sample b / rows, drawn from the stream of that sample = stream + (b / rows) * stride --
// bit-identical to S separate launches.  LRT samples differ only in their per-activation noise.  A BBB sample draws a
// whole weight tensor: the prep writes `sets` = S operand sets (tiles + bias) `set_bytes` apart in the workspace, and a
// row tile, which never straddles two samples, multiplies by the set of its sample.  LRT: sets = 1.
// first_image: the global index of row 0 (of each sample block when folded) in a batch that is split over calls (row
// blocks of a sharded MC step): the LRT noise index counts images from there, so a block draws what the whole batch
// draws at its rows.  It moves the Philox element index only; x, y, eps and workspace indexing stay local.
struct McFold { int rows; int first_image; unsigned long long stride; int sets; size_t set_bytes; };
__device__ __forceinline__ NoiseKey sample_key(NoiseKey k, const McFold& f, int j) {
    const unsigned long long s = (((unsigned long long)k.stream_hi << 32) | k.stream_lo) + (unsigned long long)j * f.stride;
    k.stream_lo = (uint32_t)s; k.stream_hi = (uint32_t)(s >> 32);
    return k;
}
__device__ __forceinline__ NoiseKey fold_key(NoiseKey k, const McFold& f, int b, int& b_in_sample) {
    b_in_sample = b;
    if (f.rows > 0) {
        const int j = b / f.rows;
        b_in_sample = b - j * f.rows;
        k = sample_key(k, f, j);
    }
    b_in_sample += f.first_image;
    return k;
}
// operand set `j` of a BBB fold (j = 0: the set an unfolded call uses)
template <class T>
__host__ __device__ __forceinline__ T* fold_set(T* p, const McFold& f, int j) {
    return reinterpret_cast<T*>(reinterpret_cast<uintptr_t>(p) + (size_t)j * f.set_bytes);
}

// The parameter half of a tensor-core layer call, common to its three kernel pairs (TcArgs, FusedArgs, S4Args derive
// from it): what the weight-prep kernel reads and writes, and what the GEMM kernel needs of the prepared operands.
struct LayerArgs {
    Geom g;
    const float* w_mu; const float* w_rho; const float* b_mu; const float* b_rho;
    const float* eps_a; const float* eps_b;        // external eps (nullptr: in-kernel Philox)
    NoiseKey key; const unsigned long long* stream_base;
    double* kl_partials; unsigned int* kl_counter; float* kl_out;
    float prior_mu, prior_sigma;
    int sample, kl_convention, has_bias, act, variant;
    // prepared-operand workspace: operand tiles in the path's own layout, then the bias rows
    // [2][npad]: row 0 = bias (BBB: sampled; LRT: mu), row 1 = LRT sigma_b^2
    __nv_bfloat16* wtiles; float* bias_ws;
    int planes;                                    // operand planes: 2 = LRT (mu, sigma^2), else 1
    McFold fold;                                   // MC samples folded into the batch (rows = 0: off)
    long long* trace;                              // debug: per-CTA clock64 checkpoints (nullptr in production)
    long long* tl_prep; long long* tl_gemm;        // debug: timeline slots of the two launches (nullptr in production)
};

// Per-element Gaussian prior of a layer (bbb_prior, include/bbb_b200.h): device pointers in the layout of W_mu and of
// bias_mu.  The weight-prep kernels take it as a parameter of its own behind their argument struct, so the structs (and
// the parameter offsets of the GEMM kernels that share them) stay as they were; only the tensor-prior instantiations
// (template flag TP) read it, and only where they compute a KL.
// w_mask / b_mask: the layer's pruning mask (bbb_masked_prior: one byte per element of W_mu / bias_mu, 0 = pruned;
// b_mask NULL: every bias kept), read by the masked instantiations (template flag MK) only, wherever mu / rho are read.
struct PriorPtrs {
    const float* w_mu; const float* w_sigma; const float* b_mu; const float* b_sigma;
    const uint8_t* w_mask; const uint8_t* b_mask;
};

// Is element i of a masked tensor kept?  A compile-time source like the prior's: KeepAll (no mask: always, no load) or
// element i of a mask (NULL: every element kept).  A pruned element is a deterministic zero in every operand and adds
// nothing to the KL: the mask selects, so its mu / rho never reach an output, whatever they hold.
struct KeepAll {};
struct KeepAt { const uint8_t* m; size_t i; };
__device__ __forceinline__ constexpr bool kept(const KeepAll&) { return true; }
__device__ __forceinline__ bool kept(const KeepAt& k) { return !k.m || __ldg(k.m + k.i) != 0; }
template <bool MK>
__device__ __forceinline__ auto w_keep(const PriorPtrs& q, size_t i) {
    if constexpr (MK) return KeepAt{q.w_mask, i};
    else return KeepAll{};
}
template <bool MK>
__device__ __forceinline__ auto b_keep(const PriorPtrs& q, size_t n) {
    if constexpr (MK) return KeepAt{q.b_mask, n};
    else return KeepAll{};
}
// The instantiation a call of the kernels above takes: f(TP, MK) with TP = a tensor prior (q.w_mu), MK = a mask
// (q.w_mask), each a std::bool_constant
template <class F>
inline auto prior_dispatch(const PriorPtrs& q, F&& f) {
    using Y = std::true_type;
    using N = std::false_type;
    if (q.w_mask) return q.w_mu ? f(Y{}, Y{}) : f(N{}, Y{});
    return q.w_mu ? f(Y{}, N{}) : f(N{}, N{});
}

// The prior of one KL term, as a compile-time source: the scalar pair of the argument struct (desc->prior_mu /
// prior_sigma) or element i of the tensors.  prior_of() is called only where the term is computed, so either is read
// only there (reading the scalars any earlier changes the code of the scalar kernels).
template <class A> struct PriorScalar { const A& p; };
struct PriorAt { const float* mu; const float* sigma; size_t i; };
struct PriorVal { float mu, sigma; };             // tensor values a kernel already loaded (batched with mu / rho)
template <class A>
__device__ __forceinline__ float2 prior_of(const PriorScalar<A>& q) { return make_float2(q.p.prior_mu, q.p.prior_sigma); }
__device__ __forceinline__ float2 prior_of(const PriorAt& q) { return make_float2(__ldg(q.mu + q.i), __ldg(q.sigma + q.i)); }
__device__ __forceinline__ float2 prior_of(const PriorVal& q) { return make_float2(q.mu, q.sigma); }
// Weight element i / bias element n: of the tensors q (TP), else the scalar pair of the argument struct `p`
template <bool TP, class A>
__device__ __forceinline__ auto w_prior(const A& p, const PriorPtrs& q, size_t i) {
    if constexpr (TP) return PriorAt{q.w_mu, q.w_sigma, i};
    else return PriorScalar<A>{p};
}
// The same for a weight element, a tensor prior loaded right away (beside the kernel's own load of mu, so the loads are
// in flight together) instead of where the KL term is computed; nothing is read without a KL (kl_out NULL)
template <bool TP, class A>
__device__ __forceinline__ auto w_prior_now(const A& p, const PriorPtrs& q, size_t i) {
    if constexpr (TP) return p.kl_out ? PriorVal{__ldg(q.w_mu + i), __ldg(q.w_sigma + i)} : PriorVal{0.0f, 1.0f};
    else return PriorScalar<A>{p};
}
template <bool TP, class A>
__device__ __forceinline__ auto b_prior(const A& p, const PriorPtrs& q, size_t n) {
    if constexpr (TP) return PriorAt{q.b_mu, q.b_sigma, n};
    else return PriorScalar<A>{p};
}

// four normals of group g (elements 4g .. 4g+3)
__device__ __forceinline__ float4 normal4(uint64_t grp, const NoiseKey& k) {
    const uint4 r = philox4x32_10(make_uint4((uint32_t)grp, (uint32_t)(grp >> 32), k.stream_lo, k.stream_hi),
                                  make_uint2(k.seed_lo, k.seed_hi));
    float4 z;
    box_muller(r.x, r.y, z.x, z.y);
    box_muller(r.z, r.w, z.z, z.w);
    return z;
}

// the normal of one element (tiling independent: same value whoever asks).
// Deliberately NOT inlined: ~110 SASS instructions per copy, and the kernels that call it
// are instruction-cache bound when it is replicated at every unrolled call site.
__device__ __noinline__ float normal1(uint64_t idx, const NoiseKey k) {
    const uint4 r = philox4x32_10(make_uint4((uint32_t)(idx >> 2), (uint32_t)(idx >> 34), k.stream_lo, k.stream_hi),
                                  make_uint2(k.seed_lo, k.seed_hi));
    const uint32_t lane = (uint32_t)idx & 3u;
    float z0, z1;
    box_muller(lane < 2 ? r.x : r.z, lane < 2 ? r.y : r.w, z0, z1);
    return (lane & 1u) ? z1 : z0;
}

// ------------------------------------------------------- elementwise math ----
// sigma = log1p(exp(rho)) exactly as the reference writes it (no threshold).
__device__ __noinline__ float softplus_sigma(float rho) { return log1pf(expf(rho)); }

// one KL term, reference convention: metrics.py:28 with (mu_q,sig_q) = prior and
// (mu_p,sig_p) = posterior (the call-site binding, SURVEY.md D1); same op order.
__device__ __noinline__ float kl_term(float mu, float sigma, float pm, float ps, int convention) {
    if (convention == BBB_KL_REFERENCE) {
        const float a = 2.0f * logf(sigma / ps);
        const float b = ps / sigma;
        const float c = (mu - pm) / sigma;
        return 0.5f * (a - 1.0f + b * b + c * c);
    }
    const float d = mu - pm;
    return logf(ps / sigma) + (sigma * sigma + d * d) / (2.0f * ps * ps) - 0.5f;
}

// The same two functions for the weight-prep kernels, which evaluate them once per weight per forward (2.2 M weights for
// BBBAlexNet) while sharing the machine with the GEMM chain: ~3x fewer instructions.  sigma keeps log1pf (the argument
// is ~1e-2: a plain log(1 + x) would lose 4 digits); the KL term uses one reciprocal instead of three divisions and the
// MUFU logarithm, whose ~1e-6 absolute error is far inside the 1e-5 relative bar of a sum of O(1)..O(100) terms
// (checked by the KL parity tests, tests/test_gpu_parity.py).
__device__ __forceinline__ float softplus_sigma_fast(float rho) { return log1pf(__expf(rho)); }
__device__ __forceinline__ float kl_term_fast(float mu, float sigma, float pm, float ps, int convention) {
    const float inv = __frcp_rn(sigma);
    const float d = mu - pm;
    if (convention == BBB_KL_REFERENCE) {
        const float b = ps * inv, c = d * inv;
        return 0.5f * (2.0f * __logf(sigma * __frcp_rn(ps)) - 1.0f + b * b + c * c);
    }
    const float ips = __frcp_rn(ps);
    return __logf(ps * inv) + 0.5f * (sigma * sigma + d * d) * ips * ips - 0.5f;
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Block-wide double sum; result valid in thread 0.  `scratch` >= 32 doubles.
__device__ __forceinline__ double block_sum(double v, double* scratch) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    v = warp_sum(v);
    if (lane == 0) scratch[wid] = v;
    __syncthreads();
    double t = 0.0;
    if (wid == 0) {
        t = lane < nw ? scratch[lane] : 0.0;
        t = warp_sum(t);
    }
    return t;
}

// Deterministic cross-CTA finish of the KL sum: every contributing CTA publishes
// its partial; the last one to arrive adds them in index order, writes the fp32
// scalar and re-arms the counter (so the workspace stays zeroed between calls).
__device__ __forceinline__ void kl_publish(double partial, int slot, int n_slots, double* partials,
                                           unsigned int* counter, float* kl_out) {
    // called by thread 0 of a contributing CTA
    partials[slot] = partial;
    __threadfence();
    const unsigned int prev = atomicAdd(counter, 1u);
    if (prev == (unsigned int)(n_slots - 1)) {
        __threadfence();
        double t = 0.0;
        for (int i = 0; i < n_slots; ++i) t += ((volatile double*)partials)[i];
        *kl_out = (float)t;
        *counter = 0u;
    }
}


// Debug timeline (bbb_debug_set_timeline): every instrumented launch owns four 64-bit slots,
// [0] = earliest CTA entry, [1] = latest CTA exit, [2] = earliest moment a CTA got past griddepcontrol.wait (kernels
// launched with programmatic serialization enter while their predecessor still runs: [1] - [2] is the part of the
// kernel that sits on the critical path), [3] unused; %globaltimer nanoseconds.  nullptr in production.
__device__ __forceinline__ unsigned long long globaltimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
__device__ __forceinline__ void tl_enter(long long* tl, int tid = 0) {
    if (tl && threadIdx.x == tid) atomicMin((unsigned long long*)tl, globaltimer_ns());
}
__device__ __forceinline__ void tl_dep(long long* tl, int tid = 0) {
    if (tl && threadIdx.x == tid) atomicMin((unsigned long long*)tl + 2, globaltimer_ns());
}
__device__ __forceinline__ void tl_exit(long long* tl, int tid = 0) {
    if (tl && threadIdx.x == tid) atomicMax((unsigned long long*)tl + 1, globaltimer_ns());
}
}  // namespace bbb
