// Fused tensor-core (wgmma) pipeline for chains of Bayesian layers on small feature maps.
//
// Between fused layers the activation lives in HBM "tiled packed": [B/128][F/64][planes] blocks of
// 128 rows x 128 B (64 bf16 of the NHWC-flattened (pixel, channel) axis), each block already in the
// SWIZZLE_128B shared-memory image, written that way by the producing epilogue; for LRT consumers the
// element-wise square is interleaved behind every x block -- so an A (A^2) tile is ONE 16 KB cp.async.bulk
// and x^2 never has to be recomputed.
//
//  (P) tap_prep_kernel / tap_prep_conv_kernel : like weight_prep_kernel but tap-major:
//      [tap][cout block][cin block][plane][NG x 64] bf16 sub-tiles, pre-swizzled, + one zero sub-tile.
//      softplus / eps / KL exactly once per weight.
//
//  (G) tap_gemm_kernel : "conv on a small map == block-structured dense layer".
//      Rows = 128 images, K walks (input pixel, 64-channel block), each output
//      column group = (output pixel, NG output channels).  For every K step the
//      tap that links the group's output pixel to the input pixel is computed; if
//      it falls outside the kernel window the MMA (and the weight copy) is skipped
//      -- zero padding costs nothing (AlexNet conv3-5: 4 of 9 taps are live).
//        warps 8-11 : producers (each owns ring stages): cp.async.bulk of A / A^2 blocks and of the
//                     live weight sub-tiles, mbarrier complete_tx
//        warps 0-7  : two warpgroups issuing wgmma (64 tile rows each, N = 64 or 128, bf16 -> fp32 in
//                     registers; LRT: 2nd accumulator), then the epilogue -- bias, sqrt(var)*eps with the
//                     LRT noise drawn in place, 2x2 max-pool across the four column groups, activation,
//                     tiled-packed bf16 (+square) or fp32 store (unpooled tiled-packed tiles: one bulk copy
//                     of the tile's shared-memory image, see tap_out_stage_bytes)
#pragma once
#include <algorithm>
#include "fwd_tc.cuh"

namespace bbb {


struct FusedArgs : LayerArgs {
    int ng, n_cblk, n_kblk, taps;
    int prev_hw;                 // linear fed by a flattened HxW map: k' = pix*C + c  <->  ref k = c*HW + pix
    const void* x; const void* x_sq;   // tiled packed input (and its square)
    void* y; void* y_sq;
    int out_mode, out_pitch, pool, in_pitch;   // pitches = F (columns) of the tiled packed matrices
    int units;                   // K blocks per pipeline step (TAP_UNITS, or 1 for the 128-column LRT tile)
};

__host__ __device__ inline size_t fused_wtile_elems(const FusedArgs& a) { return (size_t)a.planes * a.ng * 64; }
// operand sub-tiles (worst case NG=16 padding of Cout, 2 planes), the zero sub-tile (<= 2 planes x 128 rows x 128 B),
// then the bias rows
inline size_t fused_bias_offset(const Geom& g) {
    const size_t cpad = (size_t)(g.N + 63) / 64 * 64, kpad = (size_t)(g.Cin + 63) / 64 * 64;
    return cpad * kpad * g.KHW * 2 * 2 + 32768;
}
inline size_t fused_workspace_bytes(const Geom& g) { return fused_bias_offset(g) + 2 * ((size_t)(g.N + 63) / 64 * 64) * 4; }

// ------------------------------------------------------------- (P) tap prep
// Tail of both tap preps, per operand set: one all-zero sub-tile behind the real ones (staged for pool-window pixels
// whose tap is outside the kernel), then the bias rows and the KL publish.
template <bool LRT, bool FOLD, bool TP, bool MK>
__device__ __forceinline__ void tap_prep_tail(const FusedArgs& p, const PriorPtrs& q, const NoiseKey& nkey, double kl_acc) {
    const int sets = FOLD ? p.fold.sets : 1;
    const size_t sub = fused_wtile_elems(p);
    for (int j = 0; j < sets; ++j) {
        uint4* zero = reinterpret_cast<uint4*>(fold_set(p.wtiles, p.fold, j) + (size_t)p.taps * p.n_cblk * p.n_kblk * sub);
        for (long gi = (long)blockIdx.x * blockDim.x + threadIdx.x; gi < (long)(sub / 8); gi += (long)gridDim.x * blockDim.x)
            zero[gi] = make_uint4(0u, 0u, 0u, 0u);
    }
    prep_bias<LRT, FOLD, TP, MK>(p, q, nkey, p.n_cblk * p.ng, kl_acc);
    prep_finish(p, kl_acc);
}

// FOLD: BBB fold, one operand set per weight sample (a separate instantiation keeps the other preps as they were)
// Resident CTAs per SM: left to itself ptxas gives the LRT instantiation 54 registers (4 CTAs); the bound keeps it at 48
// (5 CTAs).  The other two are given the occupancy they reach anyway (40 and 64 registers): any explicit bound changes
// ptxas's register target for every instantiation of the template.
// TP: the KL is taken against the tensor prior q (bbb_prior), in the same order (both tap preps).  MK: q.w_mask /
// q.b_mask prune (both tap preps).
template <int VARIANT, bool FOLD = false, bool TP = false, bool MK = false>
__global__ void __launch_bounds__(256, VARIANT == BBB_VARIANT_LRT ? 5 : FOLD ? 4 : 6)
tap_prep_kernel(const FusedArgs p, const PriorPtrs q) {
    constexpr bool LRT = VARIANT == BBB_VARIANT_LRT;
    const Geom& g = p.g;
    const NoiseKey nkey = effective_key(p.key, p.stream_base);
    const int cprev = g.Cin / p.prev_hw;
    const size_t sub = fused_wtile_elems(p);
    const int per_sub = p.ng * 8;                                  // (row, 8-wide K chunk) items per sub-tile
    const long n_items = (long)p.taps * p.n_cblk * p.n_kblk * per_sub;
    const int sets = FOLD ? p.fold.sets : 1;
    double kl_acc = 0.0;
    tl_enter(p.tl_prep);
    for (long gi = (long)blockIdx.x * blockDim.x + threadIdx.x; gi < n_items; gi += (long)gridDim.x * blockDim.x) {
        const int st = (int)(gi / per_sub), item = (int)(gi - (long)st * per_sub);
        const int kb = st % p.n_kblk, cb = (st / p.n_kblk) % p.n_cblk, tap = st / (p.n_kblk * p.n_cblk);
        __nv_bfloat16* dst = p.wtiles + (size_t)st * sub;          // st == (tap*n_cblk + cb)*n_kblk + kb
        const int row = item % p.ng, chunk = item / p.ng;
        const int n = cb * p.ng + row;
        // element e of this chunk: packed input channel kq and its weight index (prev_hw > 1: reorder to the reference's)
        auto w_ok = [&](int e) { return n < g.N && kb * 64 + chunk * 8 + e < g.Cin; };
        auto w_index = [&](int e) {
            const int kq = kb * 64 + chunk * 8 + e;
            const int cin = (p.prev_hw > 1) ? ((kq % cprev) * p.prev_hw + kq / cprev) : kq;
            return (size_t)n * g.K + (size_t)cin * g.KHW + tap;
        };
        float w[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, s2[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        float mu8[8], sg8[8];                                      // kept for the other samples of a fold
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            mu8[e] = sg8[e] = 0.0f;
            if (w_ok(e)) {
                const size_t wi = w_index(e);
                const float mu = __ldg(p.w_mu + wi);
                const PrepElem o = prep_elem<LRT>(p, mu, RhoAt{p.w_rho, wi}, w_prior_now<TP>(p, q, wi), w_keep<MK>(q, wi),
                                                  p.eps_a, wi, wi, nkey, kl_acc);
                w[e] = o.w; s2[e] = o.s2; mu8[e] = o.mu; sg8[e] = o.sigma;
            }
        }
        // K-major SWIZZLE_128B image: row r = 128 contiguous bytes, its 16-byte chunk c stored at chunk (c ^ (r & 7))
        const int sw = row * 64 + ((chunk ^ (row & 7)) << 3);
        *reinterpret_cast<uint4*>(dst + sw) = pack_chunk<false>(w);
        if (p.planes == 2) *reinterpret_cast<uint4*>(dst + p.ng * 64 + sw) = pack_chunk<false>(s2);
        for (int j = 1; j < sets; ++j) {                           // the other samples' weights from the same mu / sigma
            const NoiseKey kj = sample_key(nkey, p.fold, j);
#pragma unroll
            for (int e = 0; e < 8; ++e) w[e] = w_ok(e) ? fold_draw(mu8[e], sg8[e], w_index(e), kj) : 0.0f;
            *reinterpret_cast<uint4*>(fold_set(dst, p.fold, j) + sw) = pack_chunk<false>(w);
        }
    }
    tap_prep_tail<LRT, FOLD, TP, MK>(p, q, nkey, kl_acc);
}

// ------------------------------------------------- (P2) tap prep, conv layers
// Same outputs as tap_prep_kernel for layers with a real kernel window (KHW > 1, prev_hw == 1), but reading the
// parameters the way they lie in memory.  tap_prep_kernel's work item is one 16-byte output chunk = 8 input
// channels of ONE tap, i.e. eight 4-byte loads KHW floats apart per thread and a different row per lane: every
// warp load touches 32 lines and every 32-byte sector is fetched KHW times (by KHW different CTAs).  That makes the
// preps LSU-bound, and they share the machine with the first
// GEMMs.  Here a CTA owns R output channels x one 64-input-channel block: each row's 64*KHW floats are contiguous
// in OIHW order and are read with consecutive lanes on consecutive floats; softplus / eps / KL are element-wise, so
// they are applied right there; the bf16 results go through shared memory ([plane][tap][row][cin]) and leave as the
// same pre-swizzled 16-byte chunks, 1 KB contiguous per (tap, plane).
// A BBB fold keeps the work split (so the KL sums in the same order as an unfolded call): phase 1 parks the fp32
// (mu, sigma) pairs in shared memory instead, and phase 2 draws every sample's weights from them, chunk by chunk.
constexpr int PREP2_BATCH = 4;                                     // loads in flight per thread
__host__ __device__ inline int prep2_slab(int R) { return R * 64 + 8; }   // bf16 per (plane, tap) slab; +8 keeps 16 B alignment, skews banks

template <int VARIANT, bool FOLD = false, bool TP = false, bool MK = false>
__global__ void __launch_bounds__(256)
tap_prep_conv_kernel(const FusedArgs p, const int R, const PriorPtrs q) {
    extern __shared__ __align__(16) uint8_t prep2_smem[];
    constexpr bool LRT = VARIANT == BBB_VARIANT_LRT;
    __nv_bfloat16* sm = reinterpret_cast<__nv_bfloat16*>(prep2_smem);
    float2* smf = reinterpret_cast<float2*>(prep2_smem);           // BBB fold: (mu, sigma) per element, same indexing
    const Geom& g = p.g;
    const NoiseKey nkey = effective_key(p.key, p.stream_base);
    constexpr bool fold = FOLD;
    const int KHW = g.KHW, L = 64 * KHW, PS = prep2_slab(R);
    const size_t sub = fused_wtile_elems(p);
    const int n_units = (p.n_cblk * p.ng / R) * p.n_kblk;
    const int dc = 256 / KHW, dq = 256 - dc * KHW;                  // (cin, tap) advance of a 256-element stride
    double kl_acc = 0.0;
    tl_enter(p.tl_prep);
    for (int unit = blockIdx.x; unit < n_units; unit += gridDim.x) {
        const int rb = unit / p.n_kblk, kb = unit - rb * p.n_kblk;
        const int n0 = rb * R, cin0 = kb * 64;
        const int total = R * L;
        // ---- phase 1: coalesced loads, element-wise math, bf16 into smem ----
        int cin = threadIdx.x / KHW, tap = threadIdx.x - cin * KHW, r = 0;
        while (cin >= 64) { cin -= 64; ++r; }
        for (int e0 = threadIdx.x; e0 < total; e0 += 256 * PREP2_BATCH) {
            float mu[PREP2_BATCH], rho[PREP2_BATCH];
            float pmu[PREP2_BATCH], psg[PREP2_BATCH];                 // TP: the prior, loaded in the same batch
            size_t wi[PREP2_BATCH];
            int so[PREP2_BATCH];                                    // smem offset of the element, -1: past the end
            bool ok[PREP2_BATCH];
#pragma unroll
            for (int u = 0; u < PREP2_BATCH; ++u) {
                const bool in = e0 + 256 * u < total;
                const int n = n0 + r;
                ok[u] = in && n < g.N && cin0 + cin < g.Cin;
                wi[u] = (size_t)n * g.K + (size_t)(cin0 + cin) * KHW + tap;
                so[u] = in ? tap * PS + r * 64 + cin : -1;
                mu[u] = ok[u] ? __ldg(p.w_mu + wi[u]) : 0.0f;
                rho[u] = (ok[u] && (p.sample || p.kl_out)) ? __ldg(p.w_rho + wi[u]) : 0.0f;
                if constexpr (TP) {
                    pmu[u] = (ok[u] && p.kl_out) ? __ldg(q.w_mu + wi[u]) : 0.0f;
                    psg[u] = (ok[u] && p.kl_out) ? __ldg(q.w_sigma + wi[u]) : 1.0f;
                }
                tap += dq; cin += dc;
                if (tap >= KHW) { tap -= KHW; ++cin; }
                while (cin >= 64) { cin -= 64; ++r; }
            }
            auto prior_u = [&](int u) {
                if constexpr (TP) return PriorVal{pmu[u], psg[u]};
                else return w_prior<false>(p, q, wi[u]);
            };
#pragma unroll
            for (int u = 0; u < PREP2_BATCH; ++u) {
                if (so[u] < 0) continue;
                PrepElem o = {0.0f, 0.0f, 0.0f};
                if (ok[u]) {
                    o = prep_elem<LRT, !fold>(p, mu[u], rho[u], prior_u(u), w_keep<MK>(q, wi[u]), p.eps_a, wi[u], wi[u],
                                              nkey, kl_acc);
                    if (fold) smf[so[u]] = make_float2(o.mu, o.sigma);   // every sample's weight is drawn in phase 2
                }
                if (fold) continue;
                sm[so[u]] = __float2bfloat16_rn(o.w);
                if (p.planes == 2) sm[KHW * PS + so[u]] = __float2bfloat16_rn(o.s2);
            }
        }
        __syncthreads();
        if (fold) {
            // ---- phase 2, BBB fold: every sample's chunk from the same (mu, sigma) ----
            for (int it = threadIdx.x; it < KHW * R * 8; it += 256) {
                const int chunk = it & 7, rr = (it >> 3) % R, tp = it / (8 * R);
                const float2* src = smf + (size_t)tp * PS + rr * 64 + chunk * 8;
                const int n = n0 + rr, cb = n / p.ng, row = n - cb * p.ng, c0 = cin0 + chunk * 8;
                const size_t st = ((size_t)tp * p.n_cblk + cb) * p.n_kblk + kb;
                const size_t wi0 = (size_t)n * g.K + (size_t)c0 * KHW + tp;
                __nv_bfloat16* dst = p.wtiles + st * sub + row * 64 + ((chunk ^ (row & 7)) << 3);
                for (int j = 0; j < p.fold.sets; ++j) {
                    const NoiseKey kj = sample_key(nkey, p.fold, j);
                    float w[8];
#pragma unroll
                    for (int e = 0; e < 8; ++e) {
                        const float2 ms = src[e];
                        w[e] = (n < g.N && c0 + e < g.Cin) ? fold_draw(ms.x, ms.y, wi0 + (size_t)e * KHW, kj) : 0.0f;
                    }
                    *reinterpret_cast<uint4*>(fold_set(dst, p.fold, j)) = pack_chunk<false>(w);
                }
            }
            __syncthreads();
            continue;
        }
        // ---- phase 2: 16-byte chunks (8 input channels of one tap) out, in the SW128 image order ----
        const int items = p.planes * KHW * R * 8;
        for (int it = threadIdx.x; it < items; it += 256) {
            const int chunk = it & 7, rr = (it >> 3) % R, pt = it / (8 * R);      // pt = plane*KHW + tap
            const int plane = pt / KHW, tp = pt - plane * KHW;
            const uint4 v = *reinterpret_cast<const uint4*>(sm + (size_t)pt * PS + rr * 64 + chunk * 8);
            const int n = n0 + rr, cb = n / p.ng, row = n - cb * p.ng;
            const size_t st = ((size_t)tp * p.n_cblk + cb) * p.n_kblk + kb;
            __nv_bfloat16* dst = p.wtiles + st * sub + (size_t)plane * p.ng * 64 + row * 64 + ((chunk ^ (row & 7)) << 3);
            *reinterpret_cast<uint4*>(dst) = v;
        }
        __syncthreads();
    }
    tap_prep_tail<LRT, FOLD, TP, MK>(p, q, nkey, kl_acc);
}

// ------------------------------------------------------------ wgmma helpers
// two packed bf16 -> their squares (exact product, one rounding: same value as bf16(float(x) * float(x)))
__device__ __forceinline__ uint32_t bf16x2_sq(uint32_t v) {
    __nv_bfloat162 h = *reinterpret_cast<__nv_bfloat162*>(&v);
    h = __hmul2(h, h);
    return *reinterpret_cast<uint32_t*>(&h);
}
// K-major SWIZZLE_128B wgmma descriptor: 8-row groups 1024 B apart, layout_type = 1 at [62,64)
__device__ __forceinline__ uint64_t make_smem_desc_sw128(uint32_t saddr) {
    return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}

constexpr int TAP_MAX_ITEMS = 64;       // live (input pixel, 64-channel block) pairs per tile (control block must stay < 2 KB)
constexpr int TAP_UNITS = 2;            // K blocks handled per pipeline step (one mbarrier phase)
static_assert(true, "");
struct FusedSmem {
    unsigned long long full[4], empty[4];
    uint32_t n_items, pad;
    float bias[128], bvar[128];     // this tile's output columns (BN <= 128)
    // K-loop schedule, built once per CTA: x = ipix | kb << 16, y = the four column groups' taps (0xFF = outside the
    // kernel window -> zero sub-tile).  A pipeline step covers TAP_UNITS consecutive items: the fixed cost of a stage
    // hand-off (barrier round trip + TMA issue + first-MMA start-up) is paid per STEP.
    int2 items[TAP_MAX_ITEMS];
    int taps_px[64];                // per input pixel: packed taps (staging for the schedule build)
};

// tap linking output pixel (oh,ow) with input pixel (ih,iw); -1 if outside the kernel window
__device__ __forceinline__ int tap_of(const Geom& g, int oh, int ow, int ih, int iw) {
    const int r = ih - oh * g.SH + g.PH, s = iw - ow * g.SW + g.PW;
    if ((unsigned)r < (unsigned)g.KH && (unsigned)s < (unsigned)g.KW) return r * g.KW + s;
    return -1;
}

// LRT activation noise of image b, output pixel pix, channels [n, n+4): Philox element index is
// the NHWC-flat index ((b*OHW + pix)*N + n), so four consecutive channels share one Philox call.
__device__ __forceinline__ float4 act_noise4(const NoiseKey& k, int b, int pix, int n, int OHW, int N) {
    const uint64_t o = ((uint64_t)b * OHW + pix) * N + n;
    if ((N & 3) == 0) return normal4(o >> 2, k);
    float4 z;
    z.x = normal1(o, k); z.y = normal1(o + 1, k); z.z = normal1(o + 2, k); z.w = normal1(o + 3, k);
    return z;
}

// Thread roles (384 threads): warps 0-7 = two warpgroups; warpgroup h issues the wgmma of tile rows [64h, 64h + 64)
// (fp32 accumulators in registers), then the pair runs the epilogue; warps 8-11 TMA producers (one elected thread each;
// the copies of a stage are dealt round-robin so their ~100-cycle issue costs overlap).
constexpr int TAP_THREADS = 384, TAP_NPROD = 4;

// Accumulators leave the registers through shared memory (the operand ring, free after the main loop): rows of BN + 4
// floats, [mean | variance] planes.  The epilogue stays a short rolled loop over 8-column chunks with one thread per
// image row -- a register-indexed epilogue would force full unrolling, and straight-line code that runs once per CTA is
// what the cold instruction cache punishes.  The LRT noise is drawn chunk by chunk in the epilogue.
__host__ __device__ constexpr size_t tap_acc_bytes(int bn, int planes) { return (size_t)planes * TC_BM * (bn + 4) * 4; }

// Unpooled tiled-packed output: the tile's BN/64 column blocks, each [x | x^2 for an LRT consumer] x 16 KB, are one
// contiguous stretch of y, and each block IS its shared-memory image.  The epilogue builds that image behind the staged
// accumulators and one thread writes it with a single bulk copy.  Thread-per-row 16-byte stores put every lane of a
// warp on a different 128-byte line, which made the stores the largest part of these layers' epilogue.
// Ragged last row tiles keep the direct stores (rows past the batch are never written).
inline size_t tap_out_stage_bytes(int bn, int pool, int out_mode, bool squares) {
    return (!pool && out_mode == OUT_PACKED_BF16) ? (size_t)(bn / 64) * (squares ? 2 : 1) * 16384 : 0;
}

// TWO: LRT variance plane (planes == 2), compile-time for the same reason as in gemm_tc_kernel
template <int BN, bool TWO>
__global__ void __launch_bounds__(TAP_THREADS, 1)
tap_gemm_kernel(const FusedArgs p, const int stages) {
    extern __shared__ uint8_t smem_raw[];
    constexpr uint32_t TB = BN * 128;                   // bytes of one B plane of a K block (BN rows x 64 bf16)
    const Geom& g = p.g;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int planes = TWO ? 2 : 1;                    // == p.planes
    constexpr bool two = TWO;
    const int ng = p.ng, groups = BN / ng;

    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;
    uint8_t* sm = smem_raw + (base - raw);
    FusedSmem* ctl = reinterpret_cast<FusedSmem*>(sm);
    const uint32_t tiles_off = 2048u;
    const uint32_t unit_bytes = (uint32_t)planes * (TC_A_BYTES + TB);   // one K block: [A][A^2][B planes]
    const int units = p.units;
    const uint32_t stage_bytes = (uint32_t)units * unit_bytes;
    const uint32_t a2_off = TC_A_BYTES, b_off = (uint32_t)planes * TC_A_BYTES;

    // output tile -> (pixel set, cout block)
    const int n_tile = blockIdx.x, m0 = blockIdx.y * TC_BM;
    const int cb = n_tile % p.n_cblk, pset = n_tile / p.n_cblk;
    // pixel of column group q: pool -> the q-th pixel of the 2x2 window `pset`; otherwise the single pixel `pset`
    const int win_y = p.pool ? pset / (g.OW >> 1) : 0, win_x = p.pool ? pset - win_y * (g.OW >> 1) : 0;
    auto group_pix = [&](int q, int& oh, int& ow) {
        if (p.pool) { oh = 2 * win_y + (q >> 1); ow = 2 * win_x + (q & 1); }
        else { oh = pset / g.OW; ow = pset - oh * g.OW; }
    };

    // debug trace: 128 slots per CTA -- [0,8) phase checkpoints, [8,40) MMA thread: full[s] passed at step it,
    // [48,88) producer 0: empty[s] passed at step it, [88,128) producer 0: step it issued
    long long* tr = p.trace ? p.trace + (size_t)(blockIdx.y * gridDim.x + blockIdx.x) * 128 : nullptr;
    if (tr && threadIdx.x == 0) tr[0] = clock64();
    tl_enter(p.tl_gemm);
    if (threadIdx.x == 0) {
        for (int s = 0; s < stages; ++s) {
            mbar_init(smem_u32(&ctl->full[s]), 1);
            mbar_init(smem_u32(&ctl->empty[s]), 8);           // lane 0 of each MMA warp once its wgmma retired
        }
        fence_barrier_init();
    }
    // K-loop schedule: one thread per input pixel works out the taps (integer divisions), thread 64 compacts
    if (threadIdx.x >= 128 && threadIdx.x < 128 + g.HW) {
        const int ipix = threadIdx.x - 128;
        const int ih = ipix / g.W, iw = ipix - ih * g.W;
        uint32_t taps = 0;
        for (int q = 0; q < 4; ++q) {
            int oh, ow;
            group_pix(q, oh, ow);
            const int tp = (q < groups) ? tap_of(g, oh, ow, ih, iw) : -1;
            taps |= (uint32_t)(tp >= 0 ? tp : 0xFF) << (8 * q);
        }
        ctl->taps_px[ipix] = (int)taps;
    }
    __syncthreads();
    if (threadIdx.x == 64) {
        int n = 0;
        for (int ipix = 0; ipix < g.HW; ++ipix) {
            const int taps = ctl->taps_px[ipix];
            if ((uint32_t)taps == 0xFFFFFFFFu) continue;
            for (int kb = 0; kb < p.n_kblk; ++kb) ctl->items[n++] = make_int2(ipix | (kb << 16), taps);
        }
        ctl->n_items = (uint32_t)n;
    }
    const bool philox = two && !p.eps_a;
    __syncthreads();
    if (tr && threadIdx.x == 0) tr[1] = clock64();

    const int n_items = (int)ctl->n_items;
    const int n_steps = (n_items + units - 1) / units;

    if (warp >= 8) {
        // ======================= TMA producers ==================================
        // The WHOLE warp executes the loop and the mbarrier waits; only the copies are issued by one lane.
        // (a try_wait that blocks with a single active lane can be woken late, while a fully converged warp is woken
        //  as soon as the phase flips.)
        // Issuing a stage costs one thread a chain of dependent latency (expect_tx + one cp.async.bulk per copy), so the
        // STEPS are dealt round-robin to the four producer warps: four issue chains run concurrently.
        // A producer must see EVERY phase of the stage it fills (parity waits alias after two phases), so at most
        // `stages` producers take part and producer p owns stage p (mod nprod).
        const int pid = warp - 8;
        const int nprod = min(TAP_NPROD, stages);
        pdl_wait();                                      // A / A^2 are the previous layer's output
        tl_dep(p.tl_gemm, 256);
        const size_t sub_elems = (size_t)planes * ng * 64;
        // BBB fold: the operand set of this row tile's weight sample (128 | rows, so the tile lies inside one sample)
        const __nv_bfloat16* wtiles = fold_set(p.wtiles, p.fold, p.fold.sets > 1 ? m0 / p.fold.rows : 0);
        const __nv_bfloat16* zero_tile = wtiles + (size_t)p.taps * p.n_cblk * p.n_kblk * sub_elems;
        const uint32_t gbytes = (uint32_t)ng * 128;                     // one group, one plane
        const uint32_t a_copy = (uint32_t)planes * TC_A_BYTES;
        const uint32_t unit_tx = a_copy + (uint32_t)(groups * planes) * gbytes;
        const size_t a_row0 = (size_t)blockIdx.y * (p.in_pitch >> 6);   // first 16 KB block of this row tile
#pragma unroll 1
        for (int it = pid; it < n_steps && pid < nprod; it += nprod) {
            const int s = it % stages;
            __syncwarp();
            mbar_wait(smem_u32(&ctl->empty[s]), ((uint32_t)(it / stages) & 1u) ^ 1u);
            if (tr && it < 40 && lane == 0) tr[48 + it] = clock64();
            if (lane == 0) {
                const int i0 = it * units, nu = min(units, n_items - i0);
                const uint32_t bar = smem_u32(&ctl->full[s]);
                mbar_arrive_expect_tx(bar, unit_tx * nu);
#pragma unroll 1
                for (int u = 0; u < nu; ++u) {
                    const int2 item = ctl->items[i0 + u];
                    const int ipix = item.x & 0xffff, kb = item.x >> 16;
                    const uint32_t st = base + tiles_off + (uint32_t)s * stage_bytes + (uint32_t)u * unit_bytes;
                    // x and x^2 blocks are interleaved in global memory and adjacent in the stage: one copy
                    const size_t a_blk = (a_row0 + (size_t)ipix * p.n_kblk + kb) * (size_t)(planes * 128 * 64);
                    bulk_g2s(st, reinterpret_cast<const __nv_bfloat16*>(p.x) + a_blk, a_copy, bar);
                    // weight planes: [plane][group][ng rows x 128 B] -> every plane is one BN-row SW128 tile
#pragma unroll 1
                    for (int q = 0; q < groups; ++q) {
                        const int tp = (item.y >> (8 * q)) & 0xFF;
                        const __nv_bfloat16* sp = tp != 0xFF ? wtiles + ((size_t)(tp * p.n_cblk + cb) * p.n_kblk + kb) * sub_elems : zero_tile;
                        if (groups == 1) {           // [mu | sigma^2] of the sub-tile are contiguous here and in the stage
                            bulk_g2s(st + b_off, sp, (uint32_t)planes * gbytes, bar);
                        } else {
                            bulk_g2s(st + b_off + q * gbytes, sp, gbytes, bar);
                            if (two) bulk_g2s(st + b_off + TB + q * gbytes, tp != 0xFF ? sp + ng * 64 : zero_tile, gbytes, bar);
                        }
                    }
                }
                if (tr && it < 40) tr[88 + it] = clock64();
            }
            __syncwarp();                                // stay converged: the next blocking wait must be a whole-warp wait
        }
    } else {
        // ======================= MMA + epilogue (warps 0-7) =====================
        // thread = (tile row t = image, half h).  Its columns, in chunks of 8:
        //   pool: the tile holds ng channels x the 4 pixels of a 2x2 window (column = q*ng + channel); half h owns ng/2
        //         channels = NC chunks, each present once per pixel q
        //   else: the tile's single pixel, columns h*BN/2 + k*8
        constexpr int NCH = BN / 16;                      // 8-column chunks per thread
        const int t = threadIdx.x & 127, h = threadIdx.x >> 7, b = m0 + t;
        const bool bvalid = b < g.B;
        const int nc = p.pool ? NCH / 4 : NCH;            // channel chunks this thread owns
        // chunk index k -> (channel chunk cc, pixel group q): pool: k = cc*4 + q (the four pixels of a chunk are consecutive)
        auto chunk_col = [&](int k, int& q, int& n0) {
            if (p.pool) { const int cc = k >> 2; q = k & 3; n0 = cb * ng + h * (ng >> 1) + cc * 8; return q * ng + h * (ng >> 1) + cc * 8; }
            q = 0; n0 = cb * BN + h * (BN / 2) + k * 8;
            return h * (BN / 2) + k * 8;
        };
        // (1) main loop: warpgroup h multiplies tile rows [64h, 64h + 64)
        float acc[BN / 2], acc2[BN / 2];
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) { acc[i] = 0.0f; acc2[i] = 0.0f; }
        {
            // descriptors are linear in the (address >> 4) field: build them once, add offsets per MMA
            const uint64_t dA0 = make_smem_desc_sw128(base + tiles_off + (uint32_t)h * 64u * 128u);
            const uint64_t dB0 = make_smem_desc_sw128(base + tiles_off + b_off);
            // One wgmma group per K block (item), one loop level: a runtime loop over the items of a step nested inside
            // the fence ... commit bracket makes ptxas serialize every wgmma.  After committing the first item of step
            // it, wait_group<1> leaves only that item in flight, so all of step it - 1 has retired: release its stage.
#pragma unroll 1
            for (int i = 0; i < n_items; ++i) {
                const int it = i / units, u = i - it * units, s = it % stages;
                if (u == 0) {
                    mbar_wait(smem_u32(&ctl->full[s]), (uint32_t)(it / stages) & 1u);
                    if (tr && it == 0 && threadIdx.x == 0) tr[3] = clock64();
                    if (tr && it < 32 && threadIdx.x == 0) tr[8 + it] = clock64();
                }
                const uint32_t so = ((uint32_t)s * stage_bytes + (uint32_t)u * unit_bytes) >> 4;
                const uint64_t da = dA0 + so, db = dB0 + so;
                wgmma_fence();
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const uint32_t acc_on = (i | j) ? 1u : 0u;
                    if (BN == 128) {
                        wgmma_m64n128k16_bf16(*reinterpret_cast<float (*)[64]>(acc), da + 2 * j, db + 2 * j, acc_on);
                        if (two) wgmma_m64n128k16_bf16(*reinterpret_cast<float (*)[64]>(acc2), da + (a2_off >> 4) + 2 * j, db + (TB >> 4) + 2 * j, acc_on);
                    } else {
                        wgmma_m64n64k16_bf16(*reinterpret_cast<float (*)[32]>(acc), da + 2 * j, db + 2 * j, acc_on);
                        if (two) wgmma_m64n64k16_bf16(*reinterpret_cast<float (*)[32]>(acc2), da + (a2_off >> 4) + 2 * j, db + (TB >> 4) + 2 * j, acc_on);
                    }
                }
                wgmma_commit();
                wgmma_wait<1>();
                if (u == 0 && it > 0 && lane == 0) mbar_arrive(smem_u32(&ctl->empty[(it - 1) % stages]));
            }
            wgmma_wait<0>();
            if (tr && threadIdx.x == 0) tr[4] = clock64();
        }
        // (2) accumulators -> shared memory (the ring is free: every step was consumed), bias of this tile
        pdl_wait();                                      // our output buffers may still be read by the previous step's consumer
        if (threadIdx.x < BN) {                          // bias / bias variance of this tile's columns (written by the prep
            const int c = threadIdx.x;                   // kernel, which may be the programmatic predecessor: after the wait)
            const int n = p.pool ? (cb * ng + (c % ng)) : (cb * BN + c);
            const float* bias_ws = fold_set(p.bias_ws, p.fold, p.fold.sets > 1 ? m0 / p.fold.rows : 0);
            ctl->bias[c] = bias_ws[n];
            ctl->bvar[c] = bias_ws[p.n_cblk * ng + n];
        }
        constexpr int AP = BN + 4;                       // row pitch in floats
        float* accs = reinterpret_cast<float*>(sm + tiles_off);
        bar_sync(1, 256);                                // both warpgroups' wgmma retired before the ring is overwritten
        // Dependents start here, not at kernel entry: one CTA per SM, so a dependent CTA resident early holds a whole SM
        // in griddepcontrol.wait, an SM another in-flight step could use.  The epilogue still hides the dependent's
        // prologue.  Only these threads, past the main loop, trigger (the first thread of a CTA to do so counts for it).
        pdl_trigger();
        acc_to_smem(acc, accs + h * 64 * AP, AP);
        if (two) acc_to_smem(acc2, accs + (TC_BM + h * 64) * AP, AP);
        bar_sync(1, 256);
        if (tr && threadIdx.x == 0) tr[5] = clock64();
        int b_s = b;                                     // image index inside its MC sample
        const NoiseKey nkey = fold_key(effective_key(p.key, p.stream_base), p.fold, b, b_s);
        const int ohw_out = p.pool ? (g.OHW >> 2) : g.OHW;
        (void)nc;
        const int planes_o = p.y_sq ? 2 : 1;
        // see tap_out_stage_bytes: the output image goes behind the staged accumulators
        const bool bulk_out = !p.pool && p.out_mode == OUT_PACKED_BF16 && m0 + TC_BM <= g.B;
        uint8_t* ostage = sm + tiles_off + tap_acc_bytes(BN, planes);
        float r[8];
#pragma unroll 1
        for (int k = 0; k < NCH; ++k) {
            int q, n0;
            const int c0 = chunk_col(k, q, n0);           // tile column / first output channel of this chunk
            float am[8];
            ld_row8(accs + t * AP + c0, am);
            if (two) {
                float av[8], e8[8];
                ld_row8(accs + (TC_BM + t) * AP + c0, av);
                int oh, ow;
                group_pix(q, oh, ow);
                if (philox) {
#pragma unroll
                    for (int hh = 0; hh < 2; ++hh) {
                        float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
                        if (bvalid && n0 + 4 * hh < g.N) z = act_noise4(nkey, b_s, oh * g.OW + ow, n0 + 4 * hh, g.OHW, g.N);
                        e8[4 * hh] = z.x; e8[4 * hh + 1] = z.y; e8[4 * hh + 2] = z.z; e8[4 * hh + 3] = z.w;
                    }
                } else {
#pragma unroll
                    for (int u = 0; u < 8; ++u)
                        e8[u] = (bvalid && n0 + u < g.N) ? __ldg(p.eps_a + ((size_t)b * g.N + n0 + u) * g.OHW + oh * g.OW + ow) : 0.0f;
                }
#pragma unroll
                for (int u = 0; u < 8; ++u) {
                    const float var = 1e-16f + (av[u] + ctl->bvar[c0 + u]);
                    am[u] = am[u] + ctl->bias[c0 + u] + fast_sqrt(var) * e8[u];
                }
            } else {
#pragma unroll
                for (int u = 0; u < 8; ++u) am[u] = am[u] + ctl->bias[c0 + u];
            }
            if (p.pool) {                                 // 2x2 max over the chunk's four pixels, store after the last
#pragma unroll
                for (int u = 0; u < 8; ++u) r[u] = q ? fmaxf(r[u], am[u]) : am[u];
                if (q < 3) continue;
            } else {
#pragma unroll
                for (int u = 0; u < 8; ++u) r[u] = am[u];
            }
            if (!bvalid) continue;
#pragma unroll
            for (int u = 0; u < 8; ++u) r[u] = fast_act(r[u], p.act);       // act is monotone: act(max) == max(act)
            if (p.out_mode == OUT_PACKED_BF16) {          // tiled packed (N % 64 == 0 guaranteed by the host)
                const uint4 v = make_uint4(pack_bf16(r[0], r[1]), pack_bf16(r[2], r[3]), pack_bf16(r[4], r[5]), pack_bf16(r[6], r[7]));
                uint4 v2 = v;
                if (p.y_sq)
                    v2 = make_uint4(pack_bf16(r[0] * r[0], r[1] * r[1]), pack_bf16(r[2] * r[2], r[3] * r[3]),
                                    pack_bf16(r[4] * r[4], r[5] * r[5]), pack_bf16(r[6] * r[6], r[7] * r[7]));
                if (bulk_out) {                           // block c0 / 64 of the tile, row t, 16-byte chunk swizzled as in HBM
                    uint8_t* d = ostage + (size_t)(c0 >> 6) * planes_o * 16384 + t * 128 + ((((c0 & 63) >> 3) ^ (t & 7)) << 4);
                    *reinterpret_cast<uint4*>(d) = v;
                    if (p.y_sq) *reinterpret_cast<uint4*>(d + 16384) = v2;
                    continue;
                }
                const size_t off = tiled_chunk_offset(b, pset * g.N + n0, p.out_pitch >> 6, planes_o);
                *reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(p.y) + off) = v;
                if (p.y_sq) *reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(p.y_sq) + off) = v2;
            } else {
                float* yo = reinterpret_cast<float*>(p.y);
#pragma unroll
                for (int u = 0; u < 8; ++u) {
                    const int n = n0 + u;
                    if (n < g.N) {
                        if (p.out_mode == OUT_ROWMAJOR_F32) yo[((size_t)b * ohw_out + pset) * g.N + n] = r[u];
                        else yo[((size_t)b * g.N + n) * ohw_out + pset] = r[u];
                    }
                }
            }
        }
        if (bulk_out) {
            fence_proxy_async();                          // this thread's image writes -> visible to the bulk copy
            bar_sync(1, 256);
            if (threadIdx.x == 0) {
                const size_t g0 = tiled_chunk_offset(m0, pset * g.N + cb * BN, p.out_pitch >> 6, planes_o);
                bulk_s2g(reinterpret_cast<__nv_bfloat16*>(p.y) + g0, smem_u32(ostage), (uint32_t)(BN / 64) * planes_o * 16384u);
                bulk_commit();
                bulk_wait_read();                         // the image must outlive the copy's reads
            }
        }
        if (tr && threadIdx.x == 0) tr[6] = clock64();
    }
    __syncthreads();
    if (tr && threadIdx.x == 256) tr[7] = clock64();
    tl_exit(p.tl_gemm, 256);
}

// ------------------------------------------------------------- host side
inline bool fused_supported(const Geom& g, int pool) {
    if (g.DH != 1 || g.DW != 1) return false;
    if (g.HW > 64) return false;                       // "small map" regime
    if (pool && ((g.OH & 1) || (g.OW & 1))) return false;
    if (g.Cin % 64) return false;                      // tiled packed input: whole 64-column blocks per pixel
    if ((long)g.HW * (g.Cin / 64) > TAP_MAX_ITEMS) return false;
    return true;
}

// The weight-prep launch of launch_fused (a.planes, ng, n_cblk, n_kblk and taps set); TP: the tensor-prior
// instantiations, MK: the masked ones.
template <bool TP, bool MK>
inline cudaError_t launch_tap_prep(const FusedArgs& a, const PriorPtrs& q, cudaStream_t st, int n_sm) {
    const Geom& g = a.g;
    const bool lrt = a.variant == BBB_VARIANT_LRT;
    const bool fold = !lrt && a.fold.sets > 1;    // one operand set per weight sample: same grid / R, so the same KL sum
    const long items = (long)a.taps * a.n_cblk * a.n_kblk * a.ng * 8;
    int grid = (int)((items + 255) / 256);
    if (grid > 2048) grid = 2048;
    if (grid < 1) grid = 1;
    prep_carveout<tap_prep_kernel<BBB_VARIANT_LRT, false, TP, MK>, tap_prep_kernel<BBB_VARIANT_BBB, false, TP, MK>, tap_prep_kernel<BBB_VARIANT_BBB, true, TP, MK>>();
    // conv layers: the coalesced variant (rows x 64-channel block per CTA); R = rows per CTA, shrunk until the
    // grid covers the SMs and the staging tile fits 48 KB
    static const bool prep2_on = [] { const char* e = getenv("BBB_B200_PREP2"); return !(e && e[0] == '0'); }();
    int R = 8;
    const int npad = a.n_cblk * a.ng;
    auto need = [&](int r) { return (size_t)a.planes * g.KHW * prep2_slab(r) * 2; };
    // <= 26 KB of staging per CTA: the preps run beside the GEMM chain (side streams) and must fit next to its CTAs
    constexpr size_t kPrepSmem = 26 * 1024;
    // (smaller CTAs -- >= 4 per SM -- were tried for more loads in flight: the preps then lose the scheduling race against
    //  the high-priority GEMM chain, and a late prep delays the whole step)
    while (R > 2 && ((long)(npad / R) * a.n_kblk < n_sm || need(R) > kPrepSmem)) R >>= 1;
    const bool prep2 = prep2_on && g.KHW > 1 && a.prev_hw == 1 && g.Cin % 64 == 0 && a.taps == g.KHW && need(R) <= 48 * 1024;
    if (prep2) {
        prep_carveout<tap_prep_conv_kernel<BBB_VARIANT_LRT, false, TP, MK>, tap_prep_conv_kernel<BBB_VARIANT_BBB, false, TP, MK>,
                      tap_prep_conv_kernel<BBB_VARIANT_BBB, true, TP, MK>>();
        int grid2 = (npad / R) * a.n_kblk;
        if (grid2 > 2048) grid2 = 2048;
        // a BBB fold stages fp32 (mu, sigma) pairs: 4x the bf16 slab, same R and grid as the unfolded call
        if (fold) {
            const size_t smem2 = (size_t)g.KHW * prep2_slab(R) * 8;
            const cudaError_t e2 = cudaFuncSetAttribute(tap_prep_conv_kernel<BBB_VARIANT_BBB, true, TP, MK>,
                                                        cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem2);
            if (e2 != cudaSuccess) return e2;
            tap_prep_conv_kernel<BBB_VARIANT_BBB, true, TP, MK><<<grid2, 256, smem2, st>>>(a, R, q);
        }
        else if (lrt) tap_prep_conv_kernel<BBB_VARIANT_LRT, false, TP, MK><<<grid2, 256, need(R), st>>>(a, R, q);
        else          tap_prep_conv_kernel<BBB_VARIANT_BBB, false, TP, MK><<<grid2, 256, need(R), st>>>(a, R, q);
    }
    else if (fold) tap_prep_kernel<BBB_VARIANT_BBB, true, TP, MK><<<grid, 256, 0, st>>>(a, q);
    else if (lrt)  tap_prep_kernel<BBB_VARIANT_LRT, false, TP, MK><<<grid, 256, 0, st>>>(a, q);
    else           tap_prep_kernel<BBB_VARIANT_BBB, false, TP, MK><<<grid, 256, 0, st>>>(a, q);
    return cudaGetLastError();
}

// q: the tensor prior and mask of the weight-prep kernel (all NULL: the scalar prior of `a`, no mask)
inline cudaError_t launch_fused(FusedArgs a, const void* x, const void* x_sq, cudaStream_t st, int* n_launch, const char** why,
                                bool do_prep = true, bool do_gemm = true, int n_sm = 132, bool prefer_wide = false,
                                const PriorPtrs& q = PriorPtrs{}) {
    const Geom& g = a.g;
    *n_launch = 0;
    a.planes = tc_planes(a.variant, a.sample);
    // tile width: 128 columns when Cout allows it and the grid still covers most of the machine (operand bytes per MAC,
    // see tap_gemm_kernel) -- or always when the caller keeps several steps in flight (bbb_set_wide_tiles) -- else 64.  BBB_B200_TAP_BN=64 forces the narrow tile (A/B measurements).
    const int psets = a.pool ? (g.OH / 2) * (g.OW / 2) : g.OHW;
    const int row_tiles = (g.B + TC_BM - 1) / TC_BM;
    int bn = 64;
    {
        static const int force = [] { const char* e = getenv("BBB_B200_TAP_BN"); return e ? atoi(e) : 0; }();
        const int ng128 = a.pool ? 32 : 128;
        if (g.N % ng128 == 0 && (prefer_wide || (long)psets * (g.N / ng128) * row_tiles >= (long)n_sm * 6 / 10)) bn = 128;
        if (force == 64 || force == 128) bn = (force == 128 && g.N % ng128 == 0) ? 128 : 64;
    }
    a.ng = a.pool ? bn / 4 : bn;
    a.n_cblk = (g.N + a.ng - 1) / a.ng;
    a.n_kblk = (g.Cin + 63) / 64;
    a.taps = g.KHW;
    a.x = x; a.x_sq = x_sq;
    if (do_gemm && a.planes == 2 && x_sq != (const void*)((const __nv_bfloat16*)x + 128 * 64)) {
        *why = "LRT fused layer needs the activation with interleaved x / x^2 blocks (x_sq == x + 8192 elements)";
        return cudaErrorInvalidValue;
    }
    if (do_prep) {
        // a tensor prior (set only when the call computes a KL) takes the TP instantiations, a mask the MK ones: same
        // kernels' grids and work split
        const cudaError_t e = prior_dispatch(q, [&](auto tp, auto mk) {
            return launch_tap_prep<decltype(tp)::value, decltype(mk)::value>(a, q, st, n_sm);
        });
        if (e != cudaSuccess) return e;
        *n_launch += 1;
    }
    if (!do_gemm) return cudaSuccess;
    // Configurations, one CTA per SM: two 384-thread CTAs would leave 85 registers per thread, fewer than the wgmma
    // accumulators of an LRT tile need.  BN = 64: stage = 2 K blocks, deep ring.  BN = 128: 64 KB (LRT) / 32 KB K
    // blocks, three stages.
    int stages;
    if (bn == 128) { stages = 3; a.units = a.planes == 2 ? 1 : 2; }
    else           { stages = a.planes == 2 ? 2 : 4; a.units = TAP_UNITS; }
    if (const char* e = getenv("BBB_B200_STAGES")) { const int v = atoi(e); if (v >= 2 && v <= stages) stages = v; }
    const size_t unit_bytes = (size_t)a.planes * (TC_A_BYTES + (size_t)bn * 128);
    // align slack + control/schedule + ring (which also holds the accumulators and the output image once the main loop
    // is done; BN = 128 LRT: 203,775 B, under the 227 KB limit)
    const size_t smem = 1023 + 2048 + std::max((size_t)stages * a.units * unit_bytes,
                                               tap_acc_bytes(bn, a.planes) + tap_out_stage_bytes(bn, a.pool, a.out_mode, a.y_sq != nullptr));
    dim3 grid(psets * a.n_cblk, row_tiles);
    cudaError_t e;
    auto launch = [&](auto kernel) {
        cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        cudaError_t e2 = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e2 != cudaSuccess) return e2;
        return launch_pdl(kernel, grid, dim3(TAP_THREADS), smem, st, a, stages);
    };
    if (a.planes == 2) e = bn == 128 ? launch(tap_gemm_kernel<128, true>) : launch(tap_gemm_kernel<64, true>);
    else               e = bn == 128 ? launch(tap_gemm_kernel<128, false>) : launch(tap_gemm_kernel<64, false>);
    if (e != cudaSuccess) return e;
    e = cudaGetLastError();
    if (e == cudaSuccess) *n_launch += 1;
    return e;
}

}  // namespace bbb
