// Bayesian layer forward on the Hopper tensor cores (BBB_MATH_BF16_TC / BBB_MATH_TF32_TC).
//
// Two kernels per layer call:
//
//  (P) weight_prep_kernel  -- HBM-bound, touches every parameter exactly once:
//      sigma = log1p(exp(rho)); closed-form KL reduced to one scalar; BBB: draws eps
//      (external or Philox) and forms W = mu + eps*sigma, LRT: forms (mu, sigma^2);
//      writes bf16 operand tiles to the workspace ALREADY IN the canonical wgmma
//      K-major core-matrix order, one contiguous 8 KB (BBB) / 16 KB (LRT) block per
//      (n-tile, k-block), so the GEMM kernel stages them with a single bulk-TMA copy.
//      Doing this once per weight instead of once per M-tile CTA removes a
//      (#M-tiles)x redundant softplus/Philox (64x for AlexNet conv2 at B=512).  It
//      depends on the parameters only, so in a captured graph it runs on a side
//      branch, off the activation critical path.
//
//  (G) gemm_tc_kernel  -- implicit-GEMM conv / linear on wgmma (M=128 tile, N=64):
//      warps 0-7 : gather the im2col rows of x (fp32 NCHW), convert to bf16 (LRT: also
//                  x^2), st.shared into the canonical K-major layout, fence.proxy.async,
//                  mbarrier arrive; then each warpgroup issues wgmma for its 64 rows
//                  (fp32 accumulators in registers; LRT: second accumulator for the
//                  variance path) and gathers the next k-block while it runs; finally
//                  the same warps run the epilogue (bias / sqrt(var)*eps -> store)
//      warp 8    : one elected thread stages the prepared weight tiles with
//                  cp.async.bulk (TMA, mbarrier complete_tx)
//
// Replaces layers/BBB/BBBConv.py:61-83, BBB/BBBLinear.py:54-76,
// BBB_LRT/BBBConv.py:62-87, BBB_LRT/BBBLinear.py:56-79, metrics.py:27-29.
#pragma once
#include <cuda_bf16.h>
#include <cstdlib>
#include "common.cuh"
#include "fwd_simt.cuh"   // apply_act

namespace bbb {

// wtiles: [n_tiles][k_blocks][planes][8 KB tile]  (64 rows x 8 K chunks of 16 bytes: 64 bf16 or 32 tf32 of K)
struct TcArgs : LayerArgs {
    const void* x; void* y; float* act_std;
    int act_dtype;           // BBB_DTYPE_BF16: x and y (NCHW) are bf16 (per-layer calls with bf16 operands only)
    int n_tiles, k_blocks;
    int skip_prep, prep_only;
    int tf32;                // operands as tf32 (fp32 storage, 4 elements per 16-byte K chunk, kind::tf32) instead of bf16
    int stage_x;             // stage the tile's input images in shared memory: 0 no, 1 as fp32, 2 as bf16 (half the
                             // footprint: lets two LRT CTAs share an SM; x^2 is then formed from the bf16 value)
    // fused epilogue (first layer of a fused chain): 2x2 max-pool + packed bf16 output
    void* y_sq; int out_mode, out_pitch, pool;     // out_mode: 0 packed bf16 [B,(pix,c)], 2 NCHW fp32 (default)
};

constexpr int TC_BM = 128, TC_BN = 64, TC_BK = 64;
constexpr int TC_TILE_ELEMS = TC_BN * TC_BK;                 // 4096 bf16 = 8 KB
constexpr int TC_A_BYTES = TC_BM * TC_BK * 2;                // 16 KB
constexpr int TC_B_BYTES = TC_BN * TC_BK * 2;                // 8 KB
constexpr int TC_SMEM_LIMIT = 227 * 1024;            // H100: opt-in shared memory per block
constexpr int TC_THREADS = 288;                    // 8 A-producer / MMA / epilogue warps + 1 weight-TMA warp

inline int tc_planes(int variant, int sample) { return (variant == BBB_VARIANT_LRT && sample) ? 2 : 1; }
inline size_t tc_stage_bytes(int planes) { return (size_t)planes * (TC_A_BYTES + TC_B_BYTES); }
// A K block is 8 chunks of 16 bytes per row whatever the operand type: 64 bf16 or 32 tf32 elements of K.
__host__ __device__ constexpr int tc_bk(bool tf32) { return tf32 ? TC_BK / 2 : TC_BK; }
inline int tc_kpad(const Geom& g, bool tf32 = false) { return (g.K + tc_bk(tf32) - 1) / tc_bk(tf32) * tc_bk(tf32); }
inline int tc_npad(const Geom& g) { return (g.N + TC_BN - 1) / TC_BN * TC_BN; }
inline size_t tc_fixed_smem(const Geom& g) { return 2048 /*two 1 KB alignment slacks*/ + 1024 /*barriers + bias*/ + (size_t)tc_kpad(g) * 8; }
inline int tc_stages(const Geom& g, int planes) {
    const long avail = (long)TC_SMEM_LIMIT - (long)tc_fixed_smem(g);
    long s = avail / (long)tc_stage_bytes(planes);
    if (s > 4) s = 4;
    return (int)s;
}
// operand tiles: 2 planes x npad rows x (kpad * 2 bytes of bf16 | kpad32 * 4 bytes of tf32), then the bias rows
inline size_t tc_bias_offset(const Geom& g, bool tf32) { return (size_t)tc_npad(g) * tc_kpad(g, tf32) * (tf32 ? 8 : 4); }
inline size_t tc_workspace_bytes(const Geom& g) {
    // the tf32 layout, never smaller than the bf16 one
    return tc_bias_offset(g, true) + (size_t)2 * tc_npad(g) * 4;
}
// Shape checks only: the activation dtype does not change the tile schedule (the callers check it).
inline bool tc_supported(const Geom& g) {
    if (g.M < 1 || g.N < 1) return false;
    if (tc_stages(g, 2) < 2) return false;
    if ((long)tc_npad(g) / TC_BN * (tc_kpad(g, true) / tc_bk(true)) > 1 << 20) return false;
    if (tc_npad(g) / TC_BN > 65535) return false;      // n tiles ride on gridDim.y
    return true;
}

// ------------------------------------------------------------------ PTX helpers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred P1;\n\t"
        "WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n\t"
        "@P1 bra DONE;\n\t"
        "bra WAIT_LOOP;\n\t"
        "DONE:\n\t"
        "}" ::"r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
// shared -> global bulk copy (bulk-group completion); the source must stay untouched until bulk_wait_read()
__device__ __forceinline__ void bulk_s2g(void* dst, uint32_t src, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }

// ---- Hopper warpgroup MMA (wgmma): D[registers of the 128 threads of a warpgroup] (+)= A[smem] * B[smem], M = 64.
// Accumulator fragment of thread (warp w of the warpgroup, lane l): d[4i + {0,1}] = row 16w + l/4, columns
// 8i + 2(l%4) + {0,1}; d[4i + {2,3}] = the same columns of row 16w + l/4 + 8.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// bf16 x bf16 -> fp32, K = 16; tf32 x tf32 -> fp32, K = 8 (operands: fp32 words, the low 13 mantissa bits ignored).
// Both read two 16-byte K chunks per row: the operand byte geometry is the same for both types.
__device__ __forceinline__ void wgmma_m64n64k16_bf16(float (&d)[32], uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(accumulate));
}

__device__ __forceinline__ void wgmma_m64n128k16_bf16(float (&d)[64], uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "r"(accumulate));
}

__device__ __forceinline__ void wgmma_m64n64k8_tf32(float (&d)[32], uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(accumulate));
}

// Park a warpgroup's m64 x (2 * NR) accumulator fragment in shared memory: `tile` = row 0 of the warpgroup's 64 rows,
// rows `pitch` floats apart.  The epilogues then read whole rows (one thread per output row).
template <int NR>
__device__ __forceinline__ void acc_to_smem(const float (&d)[NR], float* tile, int pitch) {
    const int w = (threadIdx.x >> 5) & 3, l = threadIdx.x & 31;
    float* r0 = tile + (16 * w + (l >> 2)) * pitch + 2 * (l & 3);
    float* r8 = r0 + 8 * pitch;
#pragma unroll
    for (int i = 0; i < NR / 4; ++i) {
        *reinterpret_cast<float2*>(r0 + 8 * i) = make_float2(d[4 * i], d[4 * i + 1]);
        *reinterpret_cast<float2*>(r8 + 8 * i) = make_float2(d[4 * i + 2], d[4 * i + 3]);
    }
}
__device__ __forceinline__ void ld_row8(const float* p, float (&v)[8]) {
    const float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + 4);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
// named barrier over the first `n` threads of the CTA (id 0 is __syncthreads)
__device__ __forceinline__ void bar_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }

// Programmatic dependent launch: a kernel launched with the programmatic-serialization attribute may start
// while its predecessor in the stream is still running; it must execute pdl_wait() before touching anything
// the predecessor writes.  pdl_trigger() lets the successor's CTAs start filling idle SMs early.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

inline bool pdl_enabled() {
    static int v = -1;
    // on by default: inside the captured chain the next GEMM's CTAs start on idle SMs while the previous GEMM is
    // still in its epilogue, so its prologue (barriers, K schedule) is done by the time its inputs are.
    // BBB_B200_PDL=0 turns it off.
    if (v < 0) { const char* e = getenv("BBB_B200_PDL"); v = (e && e[0] == '0') ? 0 : 1; }
    return v == 1;
}
// <<<grid, block, smem, stream>>> with the programmatic-stream-serialization attribute when enabled
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = pdl_enabled() ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}

// K-major, SWIZZLE_NONE ("interleave") wgmma shared-memory matrix descriptor (sm_90):
//   [0,14)  start address >> 4        [16,30) leading-dim byte offset >> 4 (stride between
//   the two 16-byte K chunks of one MMA)  [32,46) stride-dim byte offset >> 4 (stride between
//   8-row core-matrix groups)          [49,52) base offset = 0    [62,64) layout = 0
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)(lbo_bytes >> 4) << 16) |
           ((uint64_t)(sbo_bytes >> 4) << 32);
}
// round-to-nearest tf32 (10-bit mantissa) kept in an fp32 word: the tensor core would otherwise truncate
__device__ __forceinline__ uint32_t to_tf32(float x) {
    uint32_t u;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
    return u;
}
// one 16-byte K chunk of an operand row: 8 bf16 or 4 tf32 values
template <bool TF32>
__device__ __forceinline__ uint4 pack_chunk(const float (&v)[8]) {
    if (TF32) return make_uint4(to_tf32(v[0]), to_tf32(v[1]), to_tf32(v[2]), to_tf32(v[3]));
    const __nv_bfloat162 a = __floats2bfloat162_rn(v[0], v[1]), b = __floats2bfloat162_rn(v[2], v[3]);
    const __nv_bfloat162 c = __floats2bfloat162_rn(v[4], v[5]), d = __floats2bfloat162_rn(v[6], v[7]);
    return make_uint4(*reinterpret_cast<const uint32_t*>(&a), *reinterpret_cast<const uint32_t*>(&b),
                      *reinterpret_cast<const uint32_t*>(&c), *reinterpret_cast<const uint32_t*>(&d));
}

__device__ __forceinline__ uint32_t pack_bf16(float a, float b) {
    const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&h);
}

enum { OUT_PACKED_BF16 = 0, OUT_ROWMAJOR_F32 = 1, OUT_NCHW_F32 = 2 };

// "Tiled packed" inter-layer activation: the [B, F] bf16 matrix (F = pixels x channels, F % 64 == 0) is stored as
// [B/128 row tiles][F/64 column blocks][128 rows x 128 B], every 16 KB block already in the K-major SWIZZLE_128B
// smem image -- the consumer stages an A tile with ONE 16 KB cp.async.bulk instead of a 128-row tensor-map box
// (a strided box costs a fixed latency per stage regardless of bytes).
// When a following LRT layer also needs x^2, the two planes of a block are interleaved ([block][x | x^2], 32 KB),
// so the consumer stages both with ONE bulk copy (every cp.async.bulk has a fixed issue cost).
// Offset (in elements) of the 8-element chunk holding columns [col, col+8) of row b in plane 0:
__device__ __forceinline__ size_t tiled_chunk_offset(int b, int col, int kb_total, int planes) {
    const int r = b & 127, kb = col >> 6, ch = (col & 63) >> 3;
    return ((size_t)(b >> 7) * kb_total + kb) * (size_t)(planes * 128 * 64) + (size_t)r * 64 + (size_t)((ch ^ (r & 7)) << 3);
}

// Epilogue math of the bf16 path: MUFU-based, a handful of instructions (the exact versions in
// fwd_simt.cuh cost ~100 instructions per value and the epilogue warps run at IPC ~0.25).
// |error| <= ~1e-7 absolute: far inside the bf16 rounding of the values they feed.
__device__ __forceinline__ float fast_act(float v, int act) {
    if (act == BBB_ACT_SOFTPLUS) return fmaxf(v, 0.0f) + __logf(1.0f + __expf(-fabsf(v)));   // == nn.Softplus(1, 20)
    if (act == BBB_ACT_RELU) return fmaxf(v, 0.0f);
    return v;
}
__device__ __forceinline__ float fast_sqrt(float x) {
    float r;
    asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}
// Apply the fused activation to 16 consecutive output channels [n0, n0+16) of image b at
// output position `pos` (pixel, or pooled window) and store them in the requested layout.
struct StoreCfg { void* y; void* y_sq; int out_mode, out_pitch, N, act; };
__device__ __noinline__ void store_row16(const StoreCfg p, int b, int pos, int n0, float (&v)[16], int ohw_out) {
    const int N = p.N;
#pragma unroll
    for (int j = 0; j < 16; ++j) v[j] = fast_act(v[j], p.act);
    if (p.out_mode == OUT_PACKED_BF16 && n0 + 16 <= N) {
        const size_t off = (size_t)b * p.out_pitch + (size_t)pos * N + n0;
        uint4* yo = reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(p.y) + off);
        yo[0] = make_uint4(pack_bf16(v[0], v[1]), pack_bf16(v[2], v[3]), pack_bf16(v[4], v[5]), pack_bf16(v[6], v[7]));
        yo[1] = make_uint4(pack_bf16(v[8], v[9]), pack_bf16(v[10], v[11]), pack_bf16(v[12], v[13]), pack_bf16(v[14], v[15]));
        if (p.y_sq) {
            uint4* ys = reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(p.y_sq) + off);
            ys[0] = make_uint4(pack_bf16(v[0] * v[0], v[1] * v[1]), pack_bf16(v[2] * v[2], v[3] * v[3]), pack_bf16(v[4] * v[4], v[5] * v[5]), pack_bf16(v[6] * v[6], v[7] * v[7]));
            ys[1] = make_uint4(pack_bf16(v[8] * v[8], v[9] * v[9]), pack_bf16(v[10] * v[10], v[11] * v[11]), pack_bf16(v[12] * v[12], v[13] * v[13]), pack_bf16(v[14] * v[14], v[15] * v[15]));
        }
        return;
    }
#pragma unroll 1
    for (int j = 0; j < 16; ++j) {
        const int n = n0 + j;
        if (n >= N) break;
        if (p.out_mode == OUT_PACKED_BF16) {
            const size_t o = (size_t)b * p.out_pitch + (size_t)pos * N + n;
            reinterpret_cast<__nv_bfloat16*>(p.y)[o] = __float2bfloat16_rn(v[j]);
            if (p.y_sq) reinterpret_cast<__nv_bfloat16*>(p.y_sq)[o] = __float2bfloat16_rn(v[j] * v[j]);
        } else if (p.out_mode == OUT_ROWMAJOR_F32) {
            reinterpret_cast<float*>(p.y)[((size_t)b * ohw_out + pos) * N + n] = v[j];
        } else {
            reinterpret_cast<float*>(p.y)[((size_t)b * N + n) * ohw_out + pos] = v[j];
        }
    }
}

// ------------------------------------------------ (P) shared by every prep kernel
// The parameter math of the weight-prep kernels (weight_prep_kernel here, tap_prep_kernel / tap_prep_conv_kernel in
// fused_tc.cuh, conv_s4_prep_kernel in conv_s4_tc.cuh); each kernel adds only its index mapping and tile layout.
// The KL is a per-thread double sum in the kernel's own loop order, then prep_finish: keep both, or the KL bits move.

// rho of one element: the value a kernel already loaded, or where to read it (RhoAt).  Either way it is only used, and
// a RhoAt only read, when sigma is needed: a sampling call or one that computes the KL.
struct RhoAt { const float* rho; size_t i; };
__device__ __forceinline__ float rho_of(float rho) { return rho; }
__device__ __forceinline__ float rho_of(const RhoAt& r) { return __ldg(r.rho + r.i); }

// One parameter element: sigma = softplus(rho); plane 0 = BBB mu + eps*sigma when sampling (eps: `eps[ei]` if given,
// else Philox element i), otherwise mu; plane 1 = LRT sigma^2; and its KL term against `prior` (PriorScalar / PriorAt,
// read only here) added to `kl`.
// DRAW = false leaves plane 0 at mu: a BBB fold that draws every sample later with fold_draw.
// `keep` (KeepAll / KeepAt): a pruned element is all zeros (w, s2, sigma and the mu the fold draws from) and adds no KL
// term; nothing of its mu / rho is used, and its Philox element is not drawn (every other element's is unchanged).
struct PrepElem { float w, s2, sigma, mu; };
template <bool LRT, bool DRAW = true, class Rho, class Prior, class Keep>
__device__ __forceinline__ PrepElem prep_elem(const LayerArgs& p, float mu, const Rho& rho, const Prior& prior,
                                              const Keep& keep, const float* eps, size_t ei, uint64_t i,
                                              const NoiseKey& nkey, double& kl) {
    if constexpr (!std::is_same_v<Keep, KeepAll>) {
        if (!kept(keep)) return PrepElem{0.0f, 0.0f, 0.0f, 0.0f};
    }
    const bool stoch = p.sample != 0, do_kl = p.kl_out != nullptr;
    PrepElem o = {mu, 0.0f, 0.0f, mu};
    if (stoch || do_kl) o.sigma = softplus_sigma_fast(rho_of(rho));
    if (LRT) o.s2 = o.sigma * o.sigma;
    else if (DRAW && stoch) {
        const float e_ = eps ? __ldg(eps + ei) : normal1(i, nkey);
        o.w = mu + e_ * o.sigma;
    }
    if (do_kl) {
        const float2 q = prior_of(prior);
        kl += (double)kl_term_fast(mu, o.sigma, q.x, q.y, p.kl_convention);
    }
    return o;
}

// Weight sample j of a BBB fold: the same element drawn on sample j's stream, kj = sample_key(nkey, fold, j)
__device__ __forceinline__ float fold_draw(float mu, float sigma, uint64_t i, const NoiseKey& kj) {
    return mu + normal1(i, kj) * sigma;
}

// Bias rows of every operand set: bias_ws[n] (BBB: sampled, LRT: mu) and bias_ws[npad + n] (LRT: sigma_b^2) for all npad
// padded columns, zero past N or without a bias; one thread per column, each bias KL term counted once.  Bias element n
// is Philox element N*K + n, behind the weights.  TP: the KL terms take the bias part of the tensor prior q.
// MK: q.b_mask (if any) prunes bias elements.
template <bool LRT, bool FOLD, bool TP, bool MK>
__device__ __forceinline__ void prep_bias(const LayerArgs& p, const PriorPtrs& q, const NoiseKey& nkey, int npad, double& kl) {
    const Geom& g = p.g;
    const uint64_t i0 = (uint64_t)g.N * g.K;
    for (int n = blockIdx.x * blockDim.x + threadIdx.x; n < npad; n += gridDim.x * blockDim.x) {
        const bool real = p.has_bias && n < g.N;
        PrepElem o = {0.0f, 0.0f, 0.0f, 0.0f};
        if (real) {
            const float mu = __ldg(p.b_mu + n);
            o = prep_elem<LRT>(p, mu, RhoAt{p.b_rho, (size_t)n}, b_prior<TP>(p, q, n), b_keep<MK>(q, n), p.eps_b, n,
                               i0 + n, nkey, kl);
        }
        p.bias_ws[n] = o.w;
        p.bias_ws[npad + n] = o.s2;
        if (FOLD) {
            for (int j = 1; j < p.fold.sets; ++j) {
                float* bj = fold_set(p.bias_ws, p.fold, j);
                bj[n] = real ? fold_draw(o.mu, o.sigma, i0 + n, sample_key(nkey, p.fold, j)) : 0.0f;
                bj[npad + n] = 0.0f;
            }
        }
    }
}

// End of a prep kernel: the CTA's KL partial, published in CTA order (kl_publish), then the timeline exit
__device__ __forceinline__ void prep_finish(const LayerArgs& p, double kl) {
    __shared__ double red[32];
    if (p.kl_out) {
        const double tot = block_sum(kl, red);
        if (threadIdx.x == 0) kl_publish(tot, blockIdx.x, gridDim.x, p.kl_partials, p.kl_counter, p.kl_out);
    }
    tl_exit(p.tl_prep);
}

// Prep kernels run on the same shared-memory carve-out as the GEMM kernels: an SM only changes its L1/smem split when
// idle, so prep CTAs running at the default (small-smem) split kept the first GEMM's CTAs off every SM they touched until
// their grids drained (tools/timeline.py shows the start of each GEMM).  Set once per process for the listed kernels;
// BBB_B200_PREP_CARVEOUT=0 leaves the default split.
template <auto... Kernels>
inline void prep_carveout() {
    static const bool on = [] {
        const char* e = getenv("BBB_B200_PREP_CARVEOUT");
        if (e && e[0] == '0') return false;
        (cudaFuncSetAttribute(Kernels, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared), ...);
        return true;
    }();
    (void)on;
}

// ------------------------------------------------------------ (P) weight prep
// One CTA per (n-tile, k-block) 64x64 tile (grid-stride).  256 threads: item = (row, 8-wide
// K chunk); consecutive threads take consecutive rows so the 16-byte writes are contiguous.
// FOLD: BBB fold, one operand set per weight sample, all drawn from the same (mu, sigma) in the same work split as an
// unfolded call, so the KL sums in the same order (a separate instantiation keeps the unfolded prep as it was).
// TP: the KL is taken against the tensor prior q (bbb_prior), in the same order.  MK: q.w_mask / q.b_mask prune.
template <int VARIANT, bool TF32, bool FOLD = false, bool TP = false, bool MK = false>
__global__ void __launch_bounds__(256)
weight_prep_kernel(const TcArgs p, const PriorPtrs q) {
    constexpr bool LRT = VARIANT == BBB_VARIANT_LRT;
    static_assert(!(LRT && FOLD), "a fold prep draws BBB weight samples");
    constexpr int CE = TF32 ? 4 : 8, BKE = 8 * CE;                  // elements per 16-byte chunk / per K block
    const Geom& g = p.g;
    const NoiseKey nkey = effective_key(p.key, p.stream_base);
    constexpr int PER_TILE = TC_BN * (TC_BK / 8);                   // (row, 8-wide K chunk) items per tile
    const long n_items = (long)p.n_tiles * p.k_blocks * PER_TILE;
    double kl_acc = 0.0;
    tl_enter(p.tl_prep);
    for (long gi = (long)blockIdx.x * blockDim.x + threadIdx.x; gi < n_items; gi += (long)gridDim.x * blockDim.x) {
        const int tile = (int)(gi / PER_TILE), item = (int)(gi - (long)tile * PER_TILE);
        const int nt = tile / p.k_blocks, kb = tile - nt * p.k_blocks;
        uint8_t* dst = reinterpret_cast<uint8_t*>(p.wtiles) + (size_t)tile * p.planes * TC_B_BYTES;
        const int row = item & (TC_BN - 1), chunk = item >> 6;
        const int n = nt * TC_BN + row, k0 = kb * BKE + chunk * CE;
        float w[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, s2[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        float mu8[CE], sg8[CE];                                     // FOLD: kept for the other samples' weights
#pragma unroll
        for (int e = 0; e < CE; ++e) {
            const int k = k0 + e;
            mu8[e] = sg8[e] = 0.0f;
            if (n < g.N && k < g.K) {
                const size_t wi = (size_t)n * g.K + k;
                const float mu = __ldg(p.w_mu + wi);
                const PrepElem o = prep_elem<LRT>(p, mu, RhoAt{p.w_rho, wi}, w_prior_now<TP>(p, q, wi), w_keep<MK>(q, wi),
                                                  p.eps_a, wi, wi, nkey, kl_acc);
                w[e] = o.w; s2[e] = o.s2; mu8[e] = o.mu; sg8[e] = o.sigma;
            }
        }
        // canonical K-major core-matrix order inside the 8 KB tile: chunk*1024 + row*16 bytes
        *reinterpret_cast<uint4*>(dst + chunk * (TC_BN * 16) + row * 16) = pack_chunk<TF32>(w);
        if (p.planes == 2) *reinterpret_cast<uint4*>(dst + TC_B_BYTES + chunk * (TC_BN * 16) + row * 16) = pack_chunk<TF32>(s2);
        if (FOLD) {
            for (int j = 1; j < p.fold.sets; ++j) {
                const NoiseKey kj = sample_key(nkey, p.fold, j);
#pragma unroll
                for (int e = 0; e < CE; ++e) {
                    const int k = k0 + e;
                    w[e] = (n < g.N && k < g.K) ? fold_draw(mu8[e], sg8[e], (size_t)n * g.K + k, kj) : 0.0f;
                }
                *reinterpret_cast<uint4*>(fold_set(dst, p.fold, j) + chunk * (TC_BN * 16) + row * 16) = pack_chunk<TF32>(w);
            }
        }
    }
    prep_bias<LRT, FOLD, TP, MK>(p, q, nkey, p.n_tiles * TC_BN, kl_acc);
    prep_finish(p, kl_acc);
}

// ----------------------------------------------------------------- (G) GEMM
struct TcSmem {      // barrier block at the start of dynamic smem (after 1024-alignment)
    unsigned long long full[4], empty[4];
    float bias[64], bvar[64];
};

// Largest number of images a 128-row tile can touch (rows ordered image-major).
__host__ __device__ inline int tc_tile_images(int OHW) {
    if (TC_BM % OHW == 0) return TC_BM / OHW;          // tiles start on image boundaries
    return OHW >= TC_BM ? 2 : (TC_BM + OHW - 1) / OHW + 1;
}

// TWO: the LRT variance plane (x^2 against sigma^2) is multiplied as well (planes == 2).  A compile-time flag: a runtime
// branch around the second wgmma makes ptxas serialize every wgmma of the loop.
// BF16IO: x and y are bf16 NCHW (act_dtype = BBB_DTYPE_BF16).  The operands are the bf16 values an fp32 x rounds to,
// and the epilogue rounds the same fp32 value once: everything but the loads and stores is the fp32-I/O kernel's.
template <int VARIANT, bool TF32, bool TWO, bool BF16IO = false>
__global__ void __launch_bounds__(TC_THREADS, 2)
gemm_tc_kernel(const TcArgs p, const int stages) {
    constexpr bool LRT = VARIANT == BBB_VARIANT_LRT;
    static_assert(LRT || !TWO, "only the LRT variant has a variance plane");
    static_assert(!(TF32 && BF16IO), "bf16 activations are multiplied as bf16 operands");
    constexpr int CE = TF32 ? 4 : 8, BKE = 8 * CE;                  // elements per 16-byte chunk / per K block
    extern __shared__ uint8_t smem_raw[];
    const Geom& g = p.g;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int planes = TWO ? 2 : 1;                    // == p.planes
    constexpr bool two = TWO;

    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;
    uint8_t* sm = smem_raw + (base - raw);
    TcSmem* ctl = reinterpret_cast<TcSmem*>(sm);
    int2* ktab = reinterpret_cast<int2*>(sm + 1024);
    const int kpad = p.k_blocks * BKE;
    const uint32_t tiles_off = (1024u + (uint32_t)kpad * 8u + 1023u) & ~1023u;
    const uint32_t stage_bytes = (uint32_t)planes * (TC_A_BYTES + TC_B_BYTES);
    // stage layout: [A (16K)] [A^2 (16K, LRT)] [B planes (8K each)]
    const uint32_t a_off = 0, a2_off = TC_A_BYTES, b_off = (uint32_t)planes * TC_A_BYTES;
    float* xs = reinterpret_cast<float*>(sm + tiles_off + (size_t)stages * stage_bytes);   // staged input images (stage_x)
    __nv_bfloat16* xsh = reinterpret_cast<__nv_bfloat16*>(xs);

    const int n_tile = blockIdx.y, m_tile = blockIdx.x;     // M tiles on x: gridDim.x has no 65535 limit
    const int m0 = m_tile * TC_BM, n0 = n_tile * TC_BN;
    const int rows_here = min(TC_BM, g.M - m0);             // rows of this tile (no m0 + TC_BM: M may lie near 2^31)
    const int chw = g.Cin * g.HW;
    const int img0 = m0 / g.OHW;
    // BBB fold: the operand set of this tile's weight sample ((rows * OHW) % TC_BM == 0: the tile lies inside one sample)
    const int wset = p.fold.sets > 1 ? img0 / p.fold.rows : 0;

    long long* tr = p.trace ? p.trace + (size_t)(blockIdx.y * gridDim.x + blockIdx.x) * 128 : nullptr;
    if (tr && threadIdx.x == 0) tr[0] = clock64();
    tl_enter(p.tl_gemm);
    pdl_trigger();
    // ---- one-time setup ------------------------------------------------------
    for (int k = threadIdx.x; k < kpad; k += blockDim.x) {
        int2 e;
        if (k < g.K) {
            const int c = k / g.KHW, rs = k - c * g.KHW;
            const int r = rs / g.KW, s = rs - r * g.KW;
            e.x = c * g.HW + r * g.DH * g.W + s * g.DW;
            e.y = ((r * g.DH) << 16) | (s * g.DW);
        } else { e.x = 0; e.y = 0x7fff7fff; }
        ktab[k] = e;
    }
    pdl_wait();                                         // everything below reads/writes tensors other kernels touch
    tl_dep(p.tl_gemm);
    if (p.stage_x) {
        // the tile's input images, loaded once and coalesced; the im2col gather then reads shared memory
        // (LDS latency ~30 cycles) instead of issuing 64 dependent-latency global loads per thread and k-block
        const int last = (m0 + rows_here - 1) / g.OHW;
        const int nflt = (last - img0 + 1) * chw;
        const float* src = reinterpret_cast<const float*>(p.x) + (size_t)img0 * chw;
        const bool vec = ((reinterpret_cast<uintptr_t>(src) | (uintptr_t)(nflt * 4)) & 15u) == 0;
        if (BF16IO) {                                   // bf16 input (always staged as bf16): a plain copy
            const __nv_bfloat16* hsrc = reinterpret_cast<const __nv_bfloat16*>(p.x) + (size_t)img0 * chw;
            if (((reinterpret_cast<uintptr_t>(hsrc) | (uintptr_t)(nflt * 2)) & 15u) == 0) {
                for (int i = threadIdx.x; i < (nflt >> 3); i += blockDim.x)
                    reinterpret_cast<uint4*>(xsh)[i] = __ldg(reinterpret_cast<const uint4*>(hsrc) + i);
            } else {
                for (int i = threadIdx.x; i < nflt; i += blockDim.x) xsh[i] = hsrc[i];
            }
        } else if (p.stage_x == 2) {
            if (vec) {
                for (int i = threadIdx.x; i < (nflt >> 2); i += blockDim.x) {
                    const float4 v = __ldg(reinterpret_cast<const float4*>(src) + i);
                    reinterpret_cast<uint2*>(xsh)[i] = make_uint2(pack_bf16(v.x, v.y), pack_bf16(v.z, v.w));
                }
            } else {
                for (int i = threadIdx.x; i < nflt; i += blockDim.x) xsh[i] = __float2bfloat16_rn(__ldg(src + i));
            }
        } else if (vec) {
            for (int i = threadIdx.x; i < (nflt >> 2); i += blockDim.x)
                reinterpret_cast<float4*>(xs)[i] = __ldg(reinterpret_cast<const float4*>(src) + i);
        } else {
            for (int i = threadIdx.x; i < nflt; i += blockDim.x) xs[i] = __ldg(src + i);
        }
    }
    if (threadIdx.x < 64) {
        const int npad_ = p.n_tiles * TC_BN;
        const float* bias_ws = fold_set(p.bias_ws, p.fold, wset);
        ctl->bias[threadIdx.x] = bias_ws[n0 + threadIdx.x];
        ctl->bvar[threadIdx.x] = bias_ws[npad_ + n0 + threadIdx.x];
    }
    if (threadIdx.x == 0) {
        for (int s = 0; s < stages; ++s) {
            mbar_init(smem_u32(&ctl->full[s]), 256 + 1);      // 256 A-producer threads + the TMA thread
            mbar_init(smem_u32(&ctl->empty[s]), 8);           // lane 0 of each MMA warp once its wgmma retired
        }
        fence_barrier_init();
    }
    __syncthreads();
    if (tr && threadIdx.x == 0) tr[1] = clock64();

    if (warp < 8) {
        // ================= A producers, MMA (then epilogue) ===================
        // 8 warps: thread -> (row = t & 127, half = t >> 7); a half owns 4 of the 8 K-chunks of every k-block in the
        // main loop and 32 of the 64 output columns in the epilogue.  Warpgroup wg (== half) multiplies tile rows
        // [64 wg, 64 wg + 64): its wgmma of k-block kb runs while the same threads gather k-block kb + 1.
        const int t = threadIdx.x & 127, half = threadIdx.x >> 7;   // row of the tile
        const bool mvalid = t < rows_here;
        const int m = m0 + (mvalid ? t : 0);
        int ih0 = 0, iw0 = 0; long xb = 0;
        int bimg = 0, pix = 0;
        int pwin = 0;                                  // pooled-window index (pool mode)
        if (mvalid) {
            bimg = m / g.OHW; pix = m - bimg * g.OHW;
            int oh, ow;
            if (p.pool) {                               // rows ordered (image, window, 2x2 position): a quad of lanes == one pool window
                pwin = pix >> 2;
                const int wy = pwin / (g.OW >> 1), wx = pwin - wy * (g.OW >> 1);
                oh = 2 * wy + ((pix >> 1) & 1); ow = 2 * wx + (pix & 1);
                pix = oh * g.OW + ow;
            } else { oh = pix / g.OW; ow = pix - oh * g.OW; }
            ih0 = oh * g.SH - g.PH; iw0 = ow * g.SW - g.PW;
            xb = (long)(p.stage_x ? bimg - img0 : bimg) * chw + (long)ih0 * g.W + iw0;
        }
        const float* __restrict__ xp = p.stage_x ? xs : reinterpret_cast<const float*>(p.x);
        // BF16IO: one pointer to the staged images or to x.  With it the two-plane (LRT sampling) instantiation spills a few
        // words inside the K loop (ptxas: 36 B stored, 60 B loaded; the fp32-I/O one spills 16 / 8 B too).  Branching on
        // stage_x per element instead removes the spills, but the BBB3Conv3FC B = 2048 forward then took 5.74 ms instead of
        // 3.94-4.00 ms (H100 80GB HBM3, 700 W power limit, tools/bf16_act_bench.py).
        const __nv_bfloat16* __restrict__ xhp = p.stage_x ? xsh : reinterpret_cast<const __nv_bfloat16*>(p.x);
        float acc[32], acc2[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) { acc[i] = 0.0f; acc2[i] = 0.0f; }
        for (int kb = 0; kb < p.k_blocks; ++kb) {
            const int s = kb % stages;
            const uint32_t ph = (uint32_t)(kb / stages) & 1u;
            mbar_wait(smem_u32(&ctl->empty[s]), ph ^ 1u);
            uint8_t* st = sm + tiles_off + (size_t)s * stage_bytes;
#pragma unroll 2
            for (int c8 = half * 4; c8 < half * 4 + 4; ++c8) {
                float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
                for (int e = 0; e < CE; ++e) {
                    const int2 kt = ktab[kb * BKE + c8 * CE + e];
                    const int ih = ih0 + (kt.y >> 16), iw = iw0 + (kt.y & 0xffff);
                    float val = 0.0f;
                    if (mvalid && (unsigned)ih < (unsigned)g.H && (unsigned)iw < (unsigned)g.W) {
                        if (BF16IO) val = __bfloat162float(xhp[xb + kt.x]);
                        else val = (p.stage_x == 2) ? __bfloat162float(xsh[xb + kt.x]) : xp[xb + kt.x];
                    }
                    v[e] = val;
                }
                *reinterpret_cast<uint4*>(st + a_off + c8 * (TC_BM * 16) + t * 16) = pack_chunk<TF32>(v);
                if (two) {
#pragma unroll
                    for (int e = 0; e < 8; ++e) v[e] *= v[e];
                    *reinterpret_cast<uint4*>(st + a2_off + c8 * (TC_BM * 16) + t * 16) = pack_chunk<TF32>(v);
                }
            }
            fence_proxy_async();                        // generic-proxy stores -> visible to the tensor core
            mbar_arrive(smem_u32(&ctl->full[s]));
            if (tr && threadIdx.x == 0 && kb == 0) tr[2] = clock64();
            mbar_wait(smem_u32(&ctl->full[s]), ph);     // both halves of A and the weight tile have landed
            // one MMA = two 16-byte K chunks per row (K = 16 bf16 or 8 tf32): the byte geometry is the same for both types
            const uint32_t sa = base + tiles_off + (uint32_t)s * stage_bytes + (uint32_t)half * 64u * 16u;
            const uint32_t sb = base + tiles_off + (uint32_t)s * stage_bytes + b_off;
            wgmma_fence();
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const uint32_t acc_on = (kb | j) ? 1u : 0u;
                const uint64_t da = make_smem_desc(sa + a_off + j * 2 * (TC_BM * 16), TC_BM * 16, 128);
                const uint64_t db = make_smem_desc(sb + j * 2 * (TC_BN * 16), TC_BN * 16, 128);
                if (TF32) wgmma_m64n64k8_tf32(acc, da, db, acc_on);
                else wgmma_m64n64k16_bf16(acc, da, db, acc_on);
                if (two) {
                    const uint64_t da2 = make_smem_desc(sa + a2_off + j * 2 * (TC_BM * 16), TC_BM * 16, 128);
                    const uint64_t db2 = make_smem_desc(sb + TC_B_BYTES + j * 2 * (TC_BN * 16), TC_BN * 16, 128);
                    if (TF32) wgmma_m64n64k8_tf32(acc2, da2, db2, acc_on);
                    else wgmma_m64n64k16_bf16(acc2, da2, db2, acc_on);
                }
            }
            wgmma_commit();
            wgmma_wait<1>();                            // k-block kb - 1 retired: its stage may be refilled
            if (kb > 0 && lane == 0) mbar_arrive(smem_u32(&ctl->empty[(kb - 1) % stages]));
        }
        wgmma_wait<0>();
        if (tr && threadIdx.x == 0) tr[3] = clock64();
        // accumulators -> shared memory (the operand ring is free now), one row per thread from here on
        bar_sync(1, 256);
        constexpr int AP = TC_BN + 4;                   // row pitch in floats
        float* accs = reinterpret_cast<float*>(sm + tiles_off);
        acc_to_smem(acc, accs + half * 64 * AP, AP);
        if (two) acc_to_smem(acc2, accs + (TC_BM + half * 64) * AP, AP);
        bar_sync(1, 256);

        // ================= epilogue ============================================
        // (1) LRT noise for this row, 8 columns at a time, drawn while the last MMAs drain
        const bool philox = two && !p.eps_a;
        int b_s;                                        // image index within its MC sample (== bimg unless folded)
        const NoiseKey nkey = fold_key(effective_key(p.key, p.stream_base), p.fold, bimg, b_s);
        if (tr && threadIdx.x == 0) tr[5] = clock64();
        const int ohw_out = p.pool ? (g.OHW >> 2) : g.OHW;
        const int opix = p.pool ? pwin : pix;
        const bool writer = mvalid && !(p.pool && (threadIdx.x & 3));
#pragma unroll 1
        for (int c0 = half * 32; c0 < half * 32 + 32; c0 += 8) {
            float am[8], av[8], ez[8];
            ld_row8(accs + t * AP + c0, am);
            if (two) ld_row8(accs + (TC_BM + t) * AP + c0, av);
            const int nb = n0 + c0;
            if (philox) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (mvalid && nb + 4 * h < g.N) {
                        const uint64_t o4 = ((uint64_t)b_s * g.OHW + pix) * g.N + nb + 4 * h;   // NHWC-flat element index
                        if ((g.N & 3) == 0) z = normal4(o4 >> 2, nkey);
                        else { z.x = normal1(o4, nkey); z.y = normal1(o4 + 1, nkey); z.z = normal1(o4 + 2, nkey); z.w = normal1(o4 + 3, nkey); }
                    }
                    ez[4 * h] = z.x; ez[4 * h + 1] = z.y; ez[4 * h + 2] = z.z; ez[4 * h + 3] = z.w;
                }
            }
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int n = nb + j;
                float val = -INFINITY;
                if (mvalid && n < g.N) {
                    val = am[j] + ctl->bias[c0 + j];
                    if (two) {
                        const size_t o = ((size_t)bimg * g.N + n) * g.OHW + pix;
                        const float var = 1e-16f + (av[j] + ctl->bvar[c0 + j]);
                        const float sd = p.act_std ? sqrtf(var) : fast_sqrt(var);
                        const float e_ = philox ? ez[j] : __ldg(p.eps_a + o);
                        val = val + sd * e_;
                        if (p.act_std) p.act_std[o] = sd;
                    }
                }
                if (p.pool) {                           // 2x2 max-pool across the lane quad
                    val = fmaxf(val, __shfl_xor_sync(0xffffffffu, val, 1));
                    val = fmaxf(val, __shfl_xor_sync(0xffffffffu, val, 2));
                }
                am[j] = val;
            }
            if (!writer) continue;
#pragma unroll
            for (int j = 0; j < 8; ++j) am[j] = fast_act(am[j], p.act);   // writers only; act is monotone: act(max) == max(act)
            if (p.out_mode == OUT_PACKED_BF16) {          // tiled packed (N % 64 == 0 guaranteed by the host)
                const size_t off = tiled_chunk_offset(bimg, opix * g.N + nb, p.out_pitch >> 6, p.y_sq ? 2 : 1);
                *reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(p.y) + off) =
                    make_uint4(pack_bf16(am[0], am[1]), pack_bf16(am[2], am[3]), pack_bf16(am[4], am[5]), pack_bf16(am[6], am[7]));
                if (p.y_sq)
                    *reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(p.y_sq) + off) =
                        make_uint4(pack_bf16(am[0] * am[0], am[1] * am[1]), pack_bf16(am[2] * am[2], am[3] * am[3]),
                                   pack_bf16(am[4] * am[4], am[5] * am[5]), pack_bf16(am[6] * am[6], am[7] * am[7]));
            } else {
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const int n = nb + j;
                    if (n >= g.N) continue;
                    const size_t o = ((size_t)bimg * g.N + n) * ohw_out + opix;
                    if (BF16IO) reinterpret_cast<__nv_bfloat16*>(p.y)[o] = __float2bfloat16_rn(am[j]);
                    else reinterpret_cast<float*>(p.y)[o] = am[j];
                }
            }
        }
        if (tr && threadIdx.x == 0) tr[6] = clock64();
    } else {
        // ================= weight-tile TMA ======================================
        // whole warp waits (a blocking try_wait with one active lane can be woken late), lane 0 issues
        {
            const uint32_t bytes = (uint32_t)planes * TC_B_BYTES;
            const uint8_t* src0 = reinterpret_cast<const uint8_t*>(fold_set(p.wtiles, p.fold, wset)) + (size_t)n_tile * p.k_blocks * planes * TC_B_BYTES;
            for (int kb = 0; kb < p.k_blocks; ++kb) {
                const int s = kb % stages;
                const uint32_t ph = (uint32_t)(kb / stages) & 1u;
                __syncwarp();
                mbar_wait(smem_u32(&ctl->empty[s]), ph ^ 1u);
                if (lane == 0) {
                    const uint32_t bar = smem_u32(&ctl->full[s]);
                    mbar_arrive_expect_tx(bar, bytes);
                    bulk_g2s(base + tiles_off + (uint32_t)s * stage_bytes + b_off, src0 + (size_t)kb * planes * TC_B_BYTES, bytes, bar);
                }
                __syncwarp();
            }
        }
    }
    __syncthreads();
    if (tr && threadIdx.x == 256) tr[7] = clock64();
    tl_exit(p.tl_gemm, 256);
}

template <int VARIANT, bool TF32>
inline cudaError_t launch_fwd_tc_t(TcArgs a, cudaStream_t st, int* n_launch, const PriorPtrs& q) {
    const Geom& g = a.g;
    if (!a.skip_prep) {
        const long items = (long)a.n_tiles * a.k_blocks * TC_BN * 8;
        int grid = (int)((items + 255) / 256);
        if (grid > 2048) grid = 2048;
        // A BBB fold (one operand set per weight sample) keeps the grid, so its KL sums in the unfolded call's order.
        // (For LRT both names below are the unfolded prep: only BBB has a fold instantiation.)
        // A tensor prior (set only when the call computes a KL) takes the TP instantiations, a mask the MK ones: same grid,
        // same work split.
        constexpr bool BBB = VARIANT == BBB_VARIANT_BBB;
        prior_dispatch(q, [&](auto tp, auto mk) {
            constexpr bool TP = decltype(tp)::value, MK = decltype(mk)::value;
            prep_carveout<weight_prep_kernel<VARIANT, TF32, false, TP, MK>, weight_prep_kernel<VARIANT, TF32, BBB, TP, MK>>();
            auto* prep = BBB && a.fold.sets > 1 ? weight_prep_kernel<VARIANT, TF32, BBB, TP, MK>
                                                : weight_prep_kernel<VARIANT, TF32, false, TP, MK>;
            prep<<<grid, 256, 0, st>>>(a, q);
        });
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
        *n_launch += 1;
        a.kl_out = nullptr;
    }
    if (a.prep_only) return cudaSuccess;
    int stages = tc_stages(g, a.planes);
    // short K loops (AlexNet conv1: 6 k-blocks) gain nothing from a deep ring; two stages let two CTAs share an
    // SM (2 x (2 x 48 KB) for LRT), which hides the gather latency of one CTA behind the other and halves the waves
    if (a.k_blocks <= 8 && stages > 2) stages = 2;
    // exact footprint: base-alignment slack + control/k-table (rounded to 1 KB) + ring (+ staged images)
    const size_t tiles_off = (1024 + (size_t)tc_kpad(g, TF32) * 8 + 1023) / 1024 * 1024;
    size_t smem = 1023 + tiles_off + (size_t)stages * tc_stage_bytes(a.planes);
    const size_t xs_elems = (size_t)tc_tile_images(g.OHW) * g.Cin * g.HW;
    // bf16 activations (never with tf32 operands: the caller refuses them) stage wherever fp32 ones would, always as bf16.
    // Staging by the bf16 footprint (xs_elems * 2 <= 32 KB) would stage more layers (BBB3Conv3FC conv2); it is not done:
    // its effect is unmeasured, and this way a bf16 call and an fp32 one gather the same layers from the same memory.
    const bool bf16io = !TF32 && a.act_dtype == BBB_DTYPE_BF16;
    a.stage_x = 0;
    if (xs_elems * 4 <= 32 * 1024 && smem + xs_elems * 4 <= (size_t)TC_SMEM_LIMIT) {
        a.stage_x = 1;
        // two CTAs per SM need 2 * (smem + 1 KB reserved) <= 228 KB: try the half-size bf16 staging when fp32 does not fit
        // (never for tf32 operands: the staged copy would already have lost the bits tf32 keeps)
        const size_t per_sm = 228 * 1024;
        if (!TF32 && 2 * (smem + xs_elems * 4 + 1024) > per_sm && 2 * ((smem + xs_elems * 2 + 127) / 128 * 128 + 1024) <= per_sm) a.stage_x = 2;
        if (bf16io) a.stage_x = 2;
        smem += xs_elems * (a.stage_x == 2 ? 2 : 4);
    }
    dim3 grid((g.M - 1) / TC_BM + 1, a.n_tiles);       // not (M + TC_BM - 1): M may lie near 2^31
    // (!TF32 as BF16IO: a tf32 launcher names the fp32-I/O kernel twice rather than a bf16-I/O tf32 one)
    constexpr bool LRT = VARIANT == BBB_VARIANT_LRT;
    auto* kernel = bf16io ? (a.planes == 2 ? gemm_tc_kernel<VARIANT, TF32, LRT, !TF32> : gemm_tc_kernel<VARIANT, TF32, false, !TF32>)
                          : (a.planes == 2 ? gemm_tc_kernel<VARIANT, TF32, LRT> : gemm_tc_kernel<VARIANT, TF32, false>);
    cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    e = launch_pdl(kernel, grid, dim3(TC_THREADS), smem, st, a, stages);
    if (e != cudaSuccess) return e;
    e = cudaGetLastError();
    if (e == cudaSuccess) *n_launch += 1;
    return e;
}

// q: the tensor prior and mask of the weight-prep kernel (all NULL: the scalar prior of `a`, no mask)
inline cudaError_t launch_fwd_tc(TcArgs a, cudaStream_t st, int n_sm, int* n_launch, const PriorPtrs& q = PriorPtrs{}) {
    const Geom& g = a.g;
    const bool tf32 = a.tf32 != 0;
    a.planes = tc_planes(a.variant, a.sample);
    a.n_tiles = tc_npad(g) / TC_BN;
    a.k_blocks = tc_kpad(g, tf32) / tc_bk(tf32);
    *n_launch = 0;
    (void)n_sm;
    const bool lrt = a.variant == BBB_VARIANT_LRT;
    if (tf32) return lrt ? launch_fwd_tc_t<BBB_VARIANT_LRT, true>(a, st, n_launch, q) : launch_fwd_tc_t<BBB_VARIANT_BBB, true>(a, st, n_launch, q);
    return lrt ? launch_fwd_tc_t<BBB_VARIANT_LRT, false>(a, st, n_launch, q) : launch_fwd_tc_t<BBB_VARIANT_BBB, false>(a, st, n_launch, q);
}

}  // namespace bbb
