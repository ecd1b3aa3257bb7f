// Active-learning batch selection on the device (include/bbb_b200.h, bbb_mc_prob_log / bbb_joint_entropy):
//
//  (L) mc_prob_log_kernel   -- appends every sample's probability row p_hat_s of each image of one Monte-Carlo step
//      to a pool-long probability bank, at the score log's device-resident cursor (log_claim, score_log.cuh).
//      Bank layout: bank[i][c][s] fp32, s contiguous, S_pad = S rounded up to 8 (the tf32 wgmma K step) and C_pad = the
//      next power of two >= C; the padding is zero and never written.  So the bank is the K-major B operand of (J).
//  (J) joint_entropy_kernel -- BatchBALD's scoring GEMM with the entropy in its epilogue:
//          Q[m, (i, c)] = sum_s Pt[m][s] bank[i][c][s]          (tf32 wgmma, fp32 accumulators)
//          out[i]       = sum_m omega_m (-sum_{c < C} Q log Q)   (double, in the CTA)
//      A CTA keeps one 128-column bank tile (128 / C_pad candidates) resident in shared memory and streams every 64-row
//      tile of Pt through a cp.async ring; Q never leaves the registers.
#pragma once
#include "common.cuh"
#include "fwd_tc.cuh"      // wgmma, descriptors, to_tf32
#include "mc_head.cuh"     // softplus_f
#include "score_log.cuh"   // log_claim

namespace bbb {

constexpr int PB_THREADS = 256, PB_MAX_CTAS = 1024;

struct ProbLogArgs {
    const float* logits;                        // [S, B, C]: the step's per-sample logits
    int S, B, C, S_pad, C_pad, normalized;
    float* bank; double* expected_entropy;      // [capacity][C_pad][S_pad], [capacity]
    long long capacity;
    unsigned long long* cursor;                 // [2]: next index, images dropped
};

// One warp per image, lane = sample (s = lane, lane + 32, ..): each lane forms its samples' normalisers over the C
// classes, then writes p_hat_s[c] for c = 0 .. C-1 (32 consecutive s per store: coalesced along the bank's s).
__global__ void __launch_bounds__(PB_THREADS)
mc_prob_log_kernel(const ProbLogArgs a) {
    __shared__ unsigned long long base_sh;
    if (threadIdx.x == 0) log_claim(a.cursor, a.capacity, a.B, base_sh);
    __syncthreads();
    const unsigned long long base = base_sh;
    const int lane = threadIdx.x & 31, nwarp = PB_THREADS / 32;
    for (int b = blockIdx.x * nwarp + (threadIdx.x >> 5); b < a.B; b += gridDim.x * nwarp) {
        const unsigned long long i = base + (unsigned long long)b;
        if (i >= (unsigned long long)a.capacity) break;          // rows only grow with b
        float* dst = a.bank + (size_t)i * a.C_pad * a.S_pad;
        double h = 0.0;                                          // sum over this lane's samples of H[p_hat_s]
        for (int s = lane; s < a.S; s += 32) {
            const float* row = a.logits + ((size_t)s * a.B + b) * a.C;
            float r;                                             // as the exchange: log-sum-exp, or the softplus sum
            if (a.normalized) {
                r = 0.0f;
                for (int c = 0; c < a.C; ++c) r += softplus_f(row[c]);
            } else {
                float mx = -INFINITY, se = 0.0f;
                for (int c = 0; c < a.C; ++c) mx = fmaxf(mx, row[c]);
                for (int c = 0; c < a.C; ++c) se += expf(row[c] - mx);
                r = mx + logf(se);
            }
            for (int c = 0; c < a.C; ++c) {
                const float l = row[c];
                const float p = a.normalized ? softplus_f(l) / r : expf(l - r);
                if (p > 0.0f) h -= (double)p * log((double)p);   // 0 log 0 = 0
                dst[(size_t)c * a.S_pad + s] = __uint_as_float(to_tf32(p));
            }
        }
        h = warp_sum(h);
        if (lane == 0) a.expected_entropy[i] = h / (double)a.S;
    }
}

// ---- (J) joint entropy -----------------------------------------------------------------------------------------
constexpr int JE_THREADS = 128;              // one warpgroup
constexpr int JE_BN = 128, JE_BM = 64;       // bank columns (candidate x class) per CTA, Pt rows per wgmma tile
constexpr int JE_SMEM_LIMIT = 227 * 1024;

struct JointArgs {
    const float* pt;                          // [M_pad][S_pad], M_pad = M rounded up to JE_BM, tf32 values
    const double* omega;                      // [M]
    const unsigned char* mask;                // [N] nonzero = skip (nullable)
    const float* bank;                        // [>= N][C_pad][S_pad]
    int N, S_pad, C, C_pad, M, stages;
    double* out;                              // [N]
};

// Shared memory: [bank tile: S_pad / 4 chunks x 128 rows x 16 B][stages x Pt tile: S_pad / 4 chunks x 64 rows x 16 B],
// each in the K-major SWIZZLE_NONE core-matrix order of fwd_tc.cuh: chunk k of row r at k * rows * 16 + r * 16.
inline size_t je_smem_bytes(int S_pad, int stages) {
    return 1024 + (size_t)S_pad * 4 * (JE_BN + (size_t)stages * JE_BM);
}
// two stages where they fit beside the static per-warp column sums (4 KB): up to S_pad = 216; one from 224 up
inline int je_stages(int S_pad) { return je_smem_bytes(S_pad, 2) + 4 * JE_BN * 8 <= (size_t)JE_SMEM_LIMIT ? 2 : 1; }

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool valid) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(valid ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// -q log q of one accumulator value, 0 for q <= 0 (a rounding below 0, or an exact 0)
__device__ __forceinline__ float neg_qlogq(float q) { return q > 0.0f ? -q * __logf(q) : 0.0f; }

__global__ void __launch_bounds__(JE_THREADS, 2)
joint_entropy_kernel(const JointArgs a) {
    extern __shared__ uint8_t smem_raw[];
    __shared__ double part[4][JE_BN];                       // per-warp column sums
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;
    const int kc = a.S_pad / 4;                             // 16-byte K chunks per row
    const uint32_t b_sm = base, a_sm = base + (uint32_t)kc * JE_BN * 16;
    const uint32_t a_bytes = (uint32_t)kc * JE_BM * 16;
    const int t = threadIdx.x, w = t >> 5, l = t & 31;
    const int cand = JE_BN / a.C_pad;                       // candidates per CTA
    const int i0 = blockIdx.x * cand;
    const int n_tiles = (a.M + JE_BM - 1) / JE_BM;

    // the bank tile: row r = (candidate i0 + r / C_pad, class r % C_pad); candidates past N are zero-filled
    for (int e = t; e < kc * JE_BN; e += JE_THREADS) {
        const int r = e / kc, k = e - r * kc;
        const bool ok = i0 + r / a.C_pad < a.N;
        const float* src = a.bank + ((size_t)(ok ? i0 : 0) * a.C_pad + (ok ? r : 0)) * a.S_pad + 4 * k;
        cp_async16(b_sm + (uint32_t)(k * JE_BN + r) * 16u, src, ok);
    }
    auto load_pt = [&](int tile) {
        const uint32_t dst = a_sm + (uint32_t)(tile % a.stages) * a_bytes;
        const float* src = a.pt + (size_t)tile * JE_BM * a.S_pad;
        for (int e = t; e < kc * JE_BM; e += JE_THREADS) {
            const int r = e / kc, k = e - r * kc;
            cp_async16(dst + (uint32_t)(k * JE_BM + r) * 16u, src + (size_t)r * a.S_pad + 4 * k, true);
        }
    };
    if (a.stages > 1) load_pt(0);
    cp_async_commit();                                      // group 0: the bank tile (and Pt tile 0)

    // column sums of this thread: half h, column block j, column 8j + 2(l % 4) + e; rows 16w + l/4 (+ 8)
    double cs[2][8][2];
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int j = 0; j < 8; ++j) { cs[h][j][0] = 0.0; cs[h][j][1] = 0.0; }
    bool valid[2][8][2];                                    // column holds a real class (c < C)
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e) valid[h][j][e] = ((64 * h + 8 * j + 2 * (l & 3) + e) % a.C_pad) < a.C;

    float acc0[32], acc1[32];
#pragma unroll
    for (int r = 0; r < 32; ++r) { acc0[r] = 0.0f; acc1[r] = 0.0f; }
    for (int tile = 0; tile < n_tiles; ++tile) {
        __syncthreads();                                    // the slot refilled below was read by tile - 1's wgmma
        if (a.stages > 1) {
            if (tile + 1 < n_tiles) load_pt(tile + 1);
            cp_async_commit();
            cp_async_wait<1>();                             // everything but the newest group: tile `tile` is in
        } else {
            load_pt(tile);
            cp_async_commit();
            cp_async_wait<0>();
        }
        fence_proxy_async();                                // cp.async (generic proxy) writes -> the tensor core
        __syncthreads();
        const uint32_t sa = a_sm + (uint32_t)(tile % a.stages) * a_bytes;
        wgmma_fence();
        for (int j = 0; j < kc / 2; ++j) {                  // K = 8 per wgmma: two 16-byte chunks
            const uint64_t da = make_smem_desc(sa + (uint32_t)j * 2u * JE_BM * 16u, JE_BM * 16, 128);
            const uint64_t db0 = make_smem_desc(b_sm + (uint32_t)j * 2u * JE_BN * 16u, JE_BN * 16, 128);
            const uint64_t db1 = make_smem_desc(b_sm + (uint32_t)j * 2u * JE_BN * 16u + 64u * 16u, JE_BN * 16, 128);
            wgmma_m64n64k8_tf32(acc0, da, db0, j > 0 ? 1u : 0u);
            wgmma_m64n64k8_tf32(acc1, da, db1, j > 0 ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        const int m0 = tile * JE_BM + 16 * w + (l >> 2), m1 = m0 + 8;
        const double w0 = m0 < a.M ? __ldg(a.omega + m0) : 0.0, w1 = m1 < a.M ? __ldg(a.omega + m1) : 0.0;
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                if (valid[0][j][e])
                    cs[0][j][e] += w0 * (double)neg_qlogq(acc0[4 * j + e]) + w1 * (double)neg_qlogq(acc0[4 * j + 2 + e]);
                if (valid[1][j][e])
                    cs[1][j][e] += w0 * (double)neg_qlogq(acc1[4 * j + e]) + w1 * (double)neg_qlogq(acc1[4 * j + 2 + e]);
            }
    }
    // the 8 row groups of a warp (lanes l, l ^ 4, l ^ 8, ..), then the 4 warps, then the classes: a fixed order
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                double v = cs[h][j][e];
#pragma unroll
                for (int o = 4; o < 32; o <<= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
                if (l < 4) part[w][64 * h + 8 * j + 2 * l + e] = v;
            }
    __syncthreads();
    if (t < cand && i0 + t < a.N) {
        const int i = i0 + t;
        double s = 0.0;
        for (int c = 0; c < a.C; ++c) {
            const int col = t * a.C_pad + c;
            s += ((part[0][col] + part[1][col]) + part[2][col]) + part[3][col];
        }
        a.out[i] = (a.mask && a.mask[i]) ? -INFINITY : s;
    }
}

}  // namespace bbb
