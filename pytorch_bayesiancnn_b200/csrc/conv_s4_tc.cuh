// First-layer kernel of the fused chain: a stride-4 Bayesian conv on an NCHW fp32 image with <= 4 input channels
// (BBBAlexNet conv1: 3 -> 64, 11x11, stride 4, pad 5 -- BayesianAlexNet.py:34; forward of
// layers/BBB_LRT/BBBConv.py:62-81 / layers/BBB/BBBConv.py:61-77) with the model file's activation and 2x2/2 max-pool
// (BayesianAlexNet.py:35-36) fused, writing the tiled-packed bf16 activation (+ its square) the next layer's TMA reads.
//
// No im2col gather.  The tile's images are staged ONCE in shared memory as zero-haloed NHWC4 bf16 rows
// (pixel = 4 channels = 8 B; the x^2 plane beside it) and the tensor core reads its A operand STRAIGHT from that image:
// with stride 4 two neighbouring output pixels are 4 input pixels = 32 B apart, which is exactly the row pitch of the
// K-major SWIZZLE_32B canonical layout, so an M=128 x K=16 operand (16 images x 8 output columns; 4 input pixels x 4
// channels) is ONE shared-memory descriptor: start = (kernel row, 4-pixel group), 8-row-group stride = image pitch.
// The windows of neighbouring output pixels overlap in memory; that is fine because the hardware applies the swizzle
// XOR to the absolute shared-memory address (the bf16 parity tests of the fused chain check it), so the image
// is simply stored at swizzle(address).  K order = (kernel row r, window pixel j = s+1, channel c): per kernel row 12
// pixels x 4 channels = 48 = three K16 MMAs, the padding slots (s = -1, c = 3) carry zero weights.
//
//   CTA  = 16 images x one PAIR of output rows (2*ohp, 2*ohp+1) x all 8 output columns x 64 output channels:
//          four accumulators [row of the pair][mean | variance] x 64 columns; both rows of a pool window live in
//          the same CTA, and the weight stages are used twice.  grid = ceil(B/16) x OH/2 (AlexNet B=512: 128 CTAs).
//   warps 0-7 : stage the images (coalesced float4 loads, bf16 x and x^2, swizzled 16-byte stores); then warpgroup h
//               issues the wgmma of tile rows [64h, 64h + 64) = images [8h, 8h + 8) (12 per kernel row, fp32
//               accumulators in registers); then the epilogue through shared memory: bias, sqrt(var)*eps with the
//               LRT noise drawn in place, 2x2 max (one lane shuffle), activation, stores
//   warp 8    : weight producer: one 6/12 KB cp.async.bulk per kernel row into a 3-stage mbarrier ring
// The parameter-only half (sigma, eps, bf16 operand tiles in the K order above, KL) is conv_s4_prep_kernel.
#pragma once
#include "fused_tc.cuh"      // bf16x2_sq, tiled activation format

namespace bbb {

constexpr int S4_IMGS = 16, S4_WIN_PX = 12, S4_KROW = 48, S4_THREADS = 288;
// weight ring depth: three 12 KB stages keep the CTA at ~193 KB, so that one weight-prep CTA of a later layer (<= 26 KB,
// launch_fused) can share the SM -- with four stages every prep CTA kept a conv_s4 CTA off its SM until it had drained
constexpr int S4_STAGES = 3;
constexpr int S4_BPLANE = 64 * S4_KROW * 2;                // one plane of one kernel row: 6 chunks x 64 rows x 16 B = 6144 B

struct S4Args : LayerArgs {
    const float* x;                // a fold's x holds fold.rows images
    void* y; void* y_sq;
    int out_pitch;
    int lpad, wp, rows;            // left zero pad in pixels (PW + 1), staged row width in pixels, staged rows per image (4 + KH)
};

inline bool conv_s4_supported(const bbb_layer_desc& d, const Geom& g, int pool, int out_packed) {
    if (d.act_dtype != BBB_DTYPE_F32 || !pool || !out_packed) return false;
    if (g.Cin > 4 || g.SH != 4 || g.SW != 4 || g.DH != 1 || g.DW != 1) return false;
    if (g.OW != 8 || (g.OH & 1) || g.N != 64) return false;
    if (g.KW > S4_WIN_PX - 1 || g.KH > 16 || (g.W & 3)) return false;
    const int lpad = g.PW + 1;
    if (lpad & 1) return false;                                           // pixel pairs must stay inside one 16-byte chunk
    const int wp = max(4 * (g.OW - 1) + S4_WIN_PX, lpad + g.W);
    if (wp > 64) return false;
    const size_t img = (size_t)S4_IMGS * (4 + g.KH) * ((wp + 1) & ~1) * 8;
    return 2 * img + S4_STAGES * 2 * S4_BPLANE + 4096 <= (size_t)TC_SMEM_LIMIT;
}
// operand tiles (one 2-plane stage per kernel row), then the bias rows
inline size_t conv_s4_bias_offset(const Geom& g) { return (size_t)g.KH * 2 * S4_BPLANE; }
inline size_t conv_s4_workspace_bytes(const Geom& g) { return conv_s4_bias_offset(g) + 2 * 64 * 4 + 256; }

// ------------------------------------------------------------------ (P) prep
// item = (kernel row r, 8-wide K chunk, output channel): K' = chunk*8 + e -> window pixel j = K'/4 (s = j - 1), channel K'%4
// FOLD: BBB fold, one operand set per weight sample (a separate instantiation keeps the other preps as they were)
// TP: the KL is taken against the tensor prior q (bbb_prior), in the same order.  MK: q.w_mask / q.b_mask prune.
template <int VARIANT, bool FOLD = false, bool TP = false, bool MK = false>
__global__ void __launch_bounds__(256)
conv_s4_prep_kernel(const S4Args p, const PriorPtrs q) {
    constexpr bool LRT = VARIANT == BBB_VARIANT_LRT;
    const Geom& g = p.g;
    const int n_items = g.KH * 6 * 64;
    double kl_acc = 0.0;
    tl_enter(p.tl_prep);
    // launched with programmatic serialization in front of conv_s4_kernel: first make sure OUR predecessor (the step's
    // noise-advance kernel) is complete -- the conv kernel inherits that guarantee -- then let its CTAs start: they stage
    // their images while this kernel prepares the weights
    pdl_wait();
    pdl_trigger();
    const NoiseKey nkey = effective_key(p.key, p.stream_base);
    const int sets = FOLD ? p.fold.sets : 1;
    for (int gi = blockIdx.x * blockDim.x + threadIdx.x; gi < n_items; gi += gridDim.x * blockDim.x) {
        const int row = gi & 63, chunk = (gi >> 6) % 6, r = gi / (6 * 64);
        // weight index of element e of this chunk: window pixel s = kq / 4 - 1 (s = -1 and channel 3 are padding slots)
        auto w_ok = [&](int e) { const int kq = chunk * 8 + e, s = (kq >> 2) - 1; return s >= 0 && s < g.KW && (kq & 3) < g.Cin; };
        auto w_index = [&](int e) { const int kq = chunk * 8 + e; return (((size_t)row * g.Cin + (kq & 3)) * g.KH + r) * g.KW + (kq >> 2) - 1; };
        float w[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, s2[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        float mu8[8], sg8[8];                                       // kept for the other samples of a fold
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
        const size_t off = (size_t)r * p.planes * (S4_BPLANE / 2) + chunk * 512 + row * 8;   // canonical K-major, no swizzle
        __nv_bfloat16* dst = p.wtiles + off;
        *reinterpret_cast<uint4*>(dst) = pack_chunk<false>(w);
        if (p.planes == 2) *reinterpret_cast<uint4*>(dst + S4_BPLANE / 2) = pack_chunk<false>(s2);
        for (int j = 1; j < sets; ++j) {                            // the other samples' weights from the same mu / sigma
            const NoiseKey kj = sample_key(nkey, p.fold, j);
#pragma unroll
            for (int e = 0; e < 8; ++e) w[e] = w_ok(e) ? fold_draw(mu8[e], sg8[e], w_index(e), kj) : 0.0f;
            *reinterpret_cast<uint4*>(fold_set(p.wtiles, p.fold, j) + off) = pack_chunk<false>(w);
        }
    }
    prep_bias<LRT, FOLD, TP, MK>(p, q, nkey, 64, kl_acc);
    prep_finish(p, kl_acc);
}

// ------------------------------------------------------------------ (G) conv
struct S4Smem {
    unsigned long long full[S4_STAGES], empty[S4_STAGES], img_ready[2];
    float bias[64], bvar[64];
};

// K-major SWIZZLE_32B wgmma descriptor: rows 32 B apart, 8-row groups `sbo` bytes apart (layout type 3 at [62,64))
__device__ __forceinline__ uint64_t make_smem_desc_sw32(uint32_t saddr, uint32_t sbo_bytes) {
    return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(sbo_bytes >> 4) << 32) | (3ull << 62);
}
// shared memory of the four accumulator tiles ([row of the pair][mean | variance], 128 rows of 64 + 4 floats), staged
// over the weight ring and the images once the main loop is done
constexpr int S4_AP = 64 + 4;
__host__ __device__ constexpr size_t s4_acc_bytes(int planes) { return (size_t)2 * planes * 128 * S4_AP * 4; }
__device__ __forceinline__ uint32_t sw32(uint32_t addr) { return addr ^ (((addr >> 7) & 1u) << 4); }
template <int VARIANT>
__global__ void __launch_bounds__(S4_THREADS, 1)
conv_s4_kernel(const S4Args p) {
    constexpr bool LRT = VARIANT == BBB_VARIANT_LRT;
    extern __shared__ uint8_t smem_raw[];
    const Geom& g = p.g;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const bool two = LRT && p.planes == 2;
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;
    uint8_t* sm = smem_raw + (base - raw);
    S4Smem* ctl = reinterpret_cast<S4Smem*>(sm);
    const uint32_t stage_bytes = (uint32_t)p.planes * S4_BPLANE;
    const uint32_t ring = base + 1024u;
    const uint32_t rowb = (uint32_t)p.wp * 8u, imgb = (uint32_t)p.rows * rowb;       // bytes per staged row / image
    const uint32_t img_plane = (S4_IMGS * imgb + 127u) & ~127u;                       // + slack: windows never run past it
    const uint32_t imgx = ring + S4_STAGES * stage_bytes, imgx2 = imgx + img_plane;

    const int ohp = blockIdx.x % (g.OH >> 1), img0 = (blockIdx.x / (g.OH >> 1)) * S4_IMGS;
    const int row0 = ohp * 2 * g.SH - g.PH;                    // input row held by staged row 0

    long long* tr = p.trace ? p.trace + (size_t)blockIdx.x * 128 : nullptr;
    if (tr && threadIdx.x == 0) tr[0] = clock64();
    tl_enter(p.tl_gemm);
    if (threadIdx.x == 0) {
        for (int s = 0; s < S4_STAGES; ++s) { mbar_init(smem_u32(&ctl->full[s]), 1); mbar_init(smem_u32(&ctl->empty[s]), 8); }
        mbar_init(smem_u32(&ctl->img_ready[0]), 256);
        mbar_init(smem_u32(&ctl->img_ready[1]), 256);
        fence_barrier_init();
    }
    // No CTA-wide griddepcontrol.wait: the programmatic predecessor is this layer's weight-prep kernel (which has itself
    // waited for everything before it), and staging the images needs nothing it writes.  Only the weight producer (warp 8:
    // operand tiles, bias) and the workers' noise/epilogue (Philox base, output buffers) wait -- the image staging of all
    // CTAs overlaps the prep kernel.
    __syncthreads();
    if (tr && threadIdx.x == 0) tr[1] = clock64();

    if (warp < 8) {
        // ================= (1) stage the images ====================================================================
        // Each staging batch issues its loads for several (image, row) pairs at once, then converts and stores them.
        // The LRT noise is drawn later, in the epilogue (4).
        const int t = threadIdx.x;
        const int m = (warp & 3) * 32 + lane, half = warp >> 2;            // tile row; 32 of the 64 columns
        const int mi = m >> 3, ow = m & 7, b = img0 + mi;
        const bool bvalid = b < g.B;
        const bool philox = two && !p.eps_a;
        int b_s = b;                                                        // image index inside its MC sample
        NoiseKey nkey = p.key;                                              // completed after griddepcontrol.wait (reads the stream base)

        const int groups = g.W >> 2;                                        // float4 groups per input row
        const int n_rows = S4_IMGS * p.rows;                                // staged rows of the tile (image-major)
        const int chunks_row = p.wp >> 1, data_c0 = p.lpad >> 1, data_c1 = (p.lpad + g.W) >> 1;
        const int zc = chunks_row - (data_c1 - data_c0);                     // halo chunks per row
        const uint4 z4 = make_uint4(0u, 0u, 0u, 0u);
        auto sptr = [&](uint32_t saddr) { return reinterpret_cast<uint4*>(sm + (sw32(saddr) - base)); };   // swizzled 16-byte slot
        for (int it = t; it < n_rows * zc; it += 256) {                     // zero halo columns
            const int rowi = it / zc, k = it - rowi * zc;
            const int chunk = k < data_c0 ? k : data_c1 + (k - data_c0);
            const uint32_t off = (uint32_t)rowi * rowb + (uint32_t)chunk * 16u;
            *sptr(imgx + off) = z4;
            if (two) *sptr(imgx2 + off) = z4;
        }
        if (tr && threadIdx.x == 0) tr[40] = clock64();
        // Two batches: staged rows [0, split) first -- they are all the first kernel rows need (kernel row r reads staged
        // rows r and r + 4), so the tensor core starts on rows r < split - 4 while the second batch is still in flight.
        // thread -> (float4 group gq, slot rs); inside a batch it walks (image, row) pairs rs, rs + rstep, ... image-major
        // (consecutive slots = consecutive rows of one image = contiguous global memory; no divisions in the loop)
        const int gq = t % groups, rs = t / groups, rstep = 256 / groups;
        const size_t chw = (size_t)g.Cin * g.HW;
        const int split = min(p.rows, 2 * g.SH);
        constexpr int SB = 4;                                               // (image, row) pairs in flight per thread: 12 independent 16-byte loads
        int nit = 0;
#pragma unroll 1
        for (int batch = 0; batch < 2; ++batch) {
            const int lr0 = batch ? split : 0, nb = batch ? p.rows - split : split;   // rows of this batch
            const int n_pairs = S4_IMGS * nb;
            int pr = rs, im = nb > 0 ? rs / nb : 0, lrb = rs - im * nb;
#pragma unroll 1
            for (; pr < n_pairs; ) {
                float4 c[SB][4];
                uint32_t off[SB];
#pragma unroll
                for (int u = 0; u < SB; ++u) {
                    const int lr = lr0 + lrb, ih = row0 + lr, bb = img0 + im;
                    c[u][0] = c[u][1] = c[u][2] = c[u][3] = make_float4(0.f, 0.f, 0.f, 0.f);
                    off[u] = pr < n_pairs ? (uint32_t)(im * p.rows + lr) * rowb + (uint32_t)(p.lpad + gq * 4) * 8u : 0xffffffffu;   // 16-byte aligned: lpad even
                    if (pr < n_pairs && bb < g.B && (unsigned)ih < (unsigned)g.H) {
                        const float* src = p.x + (size_t)(p.fold.rows > 0 ? bb % p.fold.rows : bb) * chw + (size_t)ih * g.W + gq * 4;
                        c[u][0] = __ldg(reinterpret_cast<const float4*>(src));
                        if (g.Cin > 1) c[u][1] = __ldg(reinterpret_cast<const float4*>(src + g.HW));
                        if (g.Cin > 2) c[u][2] = __ldg(reinterpret_cast<const float4*>(src + 2 * g.HW));
                        if (g.Cin > 3) c[u][3] = __ldg(reinterpret_cast<const float4*>(src + 3 * g.HW));
                    }
                    pr += rstep; lrb += rstep;
                    while (lrb >= nb) { lrb -= nb; ++im; }
                }
                if (tr && threadIdx.x == 0 && nit < 2) tr[41 + 3 * nit] = clock64();
                if (tr && threadIdx.x == 0 && nit < 2) tr[42 + 3 * nit] = clock64();
#pragma unroll
                for (int u = 0; u < SB; ++u) {
                    if (off[u] == 0xffffffffu) continue;
                    const uint4 a = make_uint4(pack_bf16(c[u][0].x, c[u][1].x), pack_bf16(c[u][2].x, c[u][3].x), pack_bf16(c[u][0].y, c[u][1].y), pack_bf16(c[u][2].y, c[u][3].y));
                    const uint4 bq = make_uint4(pack_bf16(c[u][0].z, c[u][1].z), pack_bf16(c[u][2].z, c[u][3].z), pack_bf16(c[u][0].w, c[u][1].w), pack_bf16(c[u][2].w, c[u][3].w));
                    *sptr(imgx + off[u]) = a;
                    *sptr(imgx + off[u] + 16u) = bq;
                    if (two) {
                        // squares of the bf16-rounded values (what the mean path multiplies), one rounding
                        *sptr(imgx2 + off[u]) = make_uint4(bf16x2_sq(a.x), bf16x2_sq(a.y), bf16x2_sq(a.z), bf16x2_sq(a.w));
                        *sptr(imgx2 + off[u] + 16u) = make_uint4(bf16x2_sq(bq.x), bf16x2_sq(bq.y), bf16x2_sq(bq.z), bf16x2_sq(bq.w));
                    }
                }
                if (tr && threadIdx.x == 0 && nit < 2) tr[43 + 3 * nit] = clock64();
                ++nit;
            }
            fence_proxy_async();                                            // generic-proxy stores -> visible to the tensor core
            mbar_arrive(smem_u32(&ctl->img_ready[batch]));
        }
        if (tr && threadIdx.x == 0) tr[2] = clock64();
        pdl_wait();                                                         // Philox base / output buffers: everything before this launch is complete
        nkey = fold_key(effective_key(p.key, p.stream_base), p.fold, b, b_s);
        if (tr && threadIdx.x == 0) tr[3] = clock64();

        // ================= (3) MMA: warpgroup `half` owns tile rows [64 half, 64 half + 64) = images [8 half, 8 half + 8)
        // Descriptors are linear in their 16-byte address field: build the four A bases and the B base once, step them
        // by constants per kernel row, and add immediates per MMA.
        float acc[2][2][32];                                                 // [output row of the pair][mean | variance]
#pragma unroll
        for (int i = 0; i < 32; ++i) { acc[0][0][i] = 0.0f; acc[0][1][i] = 0.0f; acc[1][0][i] = 0.0f; acc[1][1][i] = 0.0f; }
        {
            const uint32_t arow_step = rowb >> 4;                            // one kernel row further down the staged image
            const uint32_t wg_off = (uint32_t)half * 8u * imgb;              // 8 images = 8 core-matrix row groups
            uint64_t dA[2][2];                                               // [output row of the pair][x | x^2], kernel row 0
#pragma unroll
            for (int ohl = 0; ohl < 2; ++ohl) {
                dA[ohl][0] = make_smem_desc_sw32(imgx + wg_off + (uint32_t)(ohl * g.SH) * rowb, imgb);
                dA[ohl][1] = make_smem_desc_sw32(imgx2 + wg_off + (uint32_t)(ohl * g.SH) * rowb, imgb);
            }
            const uint64_t dB0 = make_smem_desc(ring, 1024u, 128u);
            const int split = min(p.rows, 2 * g.SH);
            mbar_wait(smem_u32(&ctl->img_ready[0]), 0u);
#pragma unroll 1
            for (int r = 0; r < g.KH; ++r) {
                const int s = r % S4_STAGES;
                if (r + g.SH == split) mbar_wait(smem_u32(&ctl->img_ready[1]), 0u);   // staged row r + 4 belongs to the second batch
                mbar_wait(smem_u32(&ctl->full[s]), (uint32_t)(r / S4_STAGES) & 1u);
                if (tr && threadIdx.x == 0) tr[8 + r] = clock64();
                const uint64_t db = dB0 + (uint64_t)(((uint32_t)s * stage_bytes) >> 4);
                const uint32_t acc_on = r ? 1u : 0u;
                wgmma_fence();
#pragma unroll
                for (int kc = 0; kc < 3; ++kc) {
                    wgmma_m64n64k16_bf16(acc[0][0], dA[0][0] + 2 * kc, db + 128 * kc, acc_on | kc);
                    wgmma_m64n64k16_bf16(acc[1][0], dA[1][0] + 2 * kc, db + 128 * kc, acc_on | kc);
                    if (two) {
                        wgmma_m64n64k16_bf16(acc[0][1], dA[0][1] + 2 * kc, db + (S4_BPLANE >> 4) + 128 * kc, acc_on | kc);
                        wgmma_m64n64k16_bf16(acc[1][1], dA[1][1] + 2 * kc, db + (S4_BPLANE >> 4) + 128 * kc, acc_on | kc);
                    }
                }
                wgmma_commit();
                wgmma_wait<1>();                                             // kernel row r - 1 retired: its stage may be refilled
                if (r > 0 && lane == 0) mbar_arrive(smem_u32(&ctl->empty[(r - 1) % S4_STAGES]));
                dA[0][0] += arow_step; dA[0][1] += arow_step; dA[1][0] += arow_step; dA[1][1] += arow_step;
            }
            wgmma_wait<0>();
        }
        if (tr && threadIdx.x == 0) tr[4] = clock64();

        // ================= (4) epilogue ===========================================================================
        // accumulators -> shared memory over the ring and the images (both consumed), then one tile row per thread
        float* accs = reinterpret_cast<float*>(sm + (ring - base));
        bar_sync(1, 256);
        pdl_trigger();                                                      // dependents start at the epilogue (tap_gemm_kernel)
#pragma unroll
        for (int ohl = 0; ohl < 2; ++ohl) {
            acc_to_smem(acc[ohl][0], accs + ((ohl * p.planes) * 128 + half * 64) * S4_AP, S4_AP);
            if (two) acc_to_smem(acc[ohl][1], accs + ((ohl * 2 + 1) * 128 + half * 64) * S4_AP, S4_AP);
        }
        bar_sync(1, 256);
        if (tr && threadIdx.x == 0) tr[5] = clock64();
        // the other column of the 2x2 window lives in the neighbouring lane; after the shuffle both lanes hold the pooled
        // value: the even lane stores y, the odd lane y^2 (act is monotone: act(max) == max(act))
        const bool odd = ow & 1;
        const int pp = ohp * (g.OW >> 1) + (ow >> 1);
        const int kb_total = p.out_pitch >> 6, planes_out = p.y_sq ? 2 : 1;
#pragma unroll 2
        for (int c8 = 0; c8 < 4; ++c8) {                                    // 8 of this thread's 32 columns per iteration
            const int n0 = half * 32 + c8 * 8;
            float best[8];
#pragma unroll
            for (int ohl = 0; ohl < 2; ++ohl) {
                float am[8];
                ld_row8(accs + ((ohl * p.planes) * 128 + m) * S4_AP + n0, am);
                if (two) {
                    float av[8], e8[8];
                    ld_row8(accs + ((ohl * 2 + 1) * 128 + m) * S4_AP + n0, av);
                    if (philox) {
                        float4 za = make_float4(0.f, 0.f, 0.f, 0.f), zb = za;
                        if (bvalid) {
                            const uint64_t g0 = (((uint64_t)b_s * g.OHW + (uint64_t)((2 * ohp + ohl) * g.OW + ow)) * g.N + n0) >> 2;
                            za = normal4(g0, nkey); zb = normal4(g0 + 1, nkey);
                        }
                        e8[0] = za.x; e8[1] = za.y; e8[2] = za.z; e8[3] = za.w; e8[4] = zb.x; e8[5] = zb.y; e8[6] = zb.z; e8[7] = zb.w;
                    } else {
#pragma unroll
                        for (int j = 0; j < 8; ++j)
                            e8[j] = bvalid ? __ldg(p.eps_a + ((size_t)b * g.N + n0 + j) * g.OHW + (2 * ohp + ohl) * g.OW + ow) : 0.0f;
                    }
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        const float var = 1e-16f + (av[j] + ctl->bvar[n0 + j]);
                        am[j] = am[j] + ctl->bias[n0 + j] + fast_sqrt(var) * e8[j];
                    }
                } else {
#pragma unroll
                    for (int j = 0; j < 8; ++j) am[j] += ctl->bias[n0 + j];
                }
#pragma unroll
                for (int j = 0; j < 8; ++j) best[j] = ohl ? fmaxf(best[j], am[j]) : am[j];
            }
            float v[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                float q = best[j];
                q = fmaxf(q, __shfl_xor_sync(0xffffffffu, q, 1));
                q = fast_act(q, p.act);
                v[j] = odd ? q * q : q;
            }
            if (bvalid && (!odd || p.y_sq)) {
                const size_t off = tiled_chunk_offset(b, pp * g.N + n0, kb_total, planes_out);
                __nv_bfloat16* dst = reinterpret_cast<__nv_bfloat16*>(odd ? p.y_sq : p.y) + off;
                *reinterpret_cast<uint4*>(dst) = make_uint4(pack_bf16(v[0], v[1]), pack_bf16(v[2], v[3]), pack_bf16(v[4], v[5]), pack_bf16(v[6], v[7]));
            }
        }
        if (tr && threadIdx.x == 0) tr[6] = clock64();
    } else {
        // ================= weight producer ============================================================================
        pdl_wait();                                                         // the prep kernel's tiles and bias
        tl_dep(p.tl_gemm, 256);
        // BBB fold: the weight sample of this CTA's images (16 | rows, so the CTA lies inside one sample)
        const int set = p.fold.sets > 1 ? img0 / p.fold.rows : 0;
        const float* bias_ws = fold_set(p.bias_ws, p.fold, set);
        const __nv_bfloat16* wtiles = fold_set(p.wtiles, p.fold, set);
        for (int c = lane; c < 64; c += 32) {
            ctl->bias[c] = bias_ws[c];
            ctl->bvar[c] = bias_ws[64 + c];
        }
        __syncwarp();                                                       // bias stores ordered before lane 0's first mbarrier arrive
        for (int r = 0; r < g.KH; ++r) {
            const int s = r % S4_STAGES;
            __syncwarp();
            mbar_wait(smem_u32(&ctl->empty[s]), ((uint32_t)(r / S4_STAGES) & 1u) ^ 1u);
            if (lane == 0) {
                const uint32_t bar = smem_u32(&ctl->full[s]);
                mbar_arrive_expect_tx(bar, stage_bytes);
                bulk_g2s(ring + (uint32_t)s * stage_bytes, wtiles + (size_t)r * (stage_bytes / 2), stage_bytes, bar);
            }
            __syncwarp();
        }
    }
    __syncthreads();
    if (tr && threadIdx.x == 256) tr[7] = clock64();
    tl_exit(p.tl_gemm, 256);
}

// q: the tensor prior and mask of the weight-prep kernel (all NULL: the scalar prior of `a`, no mask)
inline cudaError_t launch_conv_s4(S4Args a, cudaStream_t st, bool do_prep, bool do_gemm, int* n_launch, const PriorPtrs& q = PriorPtrs{}) {
    const Geom& g = a.g;
    *n_launch = 0;
    a.planes = tc_planes(a.variant, a.sample);
    a.lpad = g.PW + 1;
    a.wp = (max(4 * (g.OW - 1) + S4_WIN_PX, a.lpad + g.W) + 1) & ~1;
    a.rows = 4 + g.KH;
    const bool lrt = a.variant == BBB_VARIANT_LRT;
    if (do_prep) {
        const int grid = (g.KH * 6 * 64 + 255) / 256;
        // a tensor prior (set only when the call computes a KL) or a mask: same grid and work split
        cudaError_t e = prior_dispatch(q, [&](auto tp, auto mk) {
            constexpr bool TP = decltype(tp)::value, MK = decltype(mk)::value;
            prep_carveout<conv_s4_prep_kernel<BBB_VARIANT_LRT, false, TP, MK>, conv_s4_prep_kernel<BBB_VARIANT_BBB, false, TP, MK>,
                          conv_s4_prep_kernel<BBB_VARIANT_BBB, true, TP, MK>>();
            return lrt ? launch_pdl(conv_s4_prep_kernel<BBB_VARIANT_LRT, false, TP, MK>, dim3(grid), dim3(256), 0, st, a, q)
                : a.fold.sets > 1 ? launch_pdl(conv_s4_prep_kernel<BBB_VARIANT_BBB, true, TP, MK>, dim3(grid), dim3(256), 0, st, a, q)
                                  : launch_pdl(conv_s4_prep_kernel<BBB_VARIANT_BBB, false, TP, MK>, dim3(grid), dim3(256), 0, st, a, q);
        });
        if (e == cudaSuccess) e = cudaGetLastError();
        if (e != cudaSuccess) return e;
        *n_launch += 1;
    }
    if (!do_gemm) return cudaSuccess;
    const size_t imgb = (size_t)a.rows * a.wp * 8, img_plane = (S4_IMGS * imgb + 127) / 128 * 128;
    const size_t smem = 1023 + 1024 + std::max((size_t)S4_STAGES * a.planes * S4_BPLANE + a.planes * img_plane + 256, s4_acc_bytes(a.planes));
    dim3 grid((unsigned)((g.B + S4_IMGS - 1) / S4_IMGS) * (g.OH >> 1));
    auto launch = [&](auto kernel) {
        cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        cudaError_t e2 = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e2 != cudaSuccess) return e2;
        return launch_pdl(kernel, grid, dim3(S4_THREADS), smem, st, a);
    };
    cudaError_t e = lrt ? launch(conv_s4_kernel<BBB_VARIANT_LRT>) : launch(conv_s4_kernel<BBB_VARIANT_BBB>);
    if (e != cudaSuccess) return e;
    e = cudaGetLastError();
    if (e == cudaSuccess) *n_launch += 1;
    return e;
}

}  // namespace bbb
