// Fused multi-head attention for the UNet's and the text encoder's transformer blocks: O = softmax(Q K^T * scale) V per
// (image, head); scores never leave the SM.  wgmma with register accumulators, TMA-fed Q / K / V^T tiles.
//
// CTA = 128 queries of one (image, head); 288 threads:
//   warps 0-3 / 4-7  two consumer warpgroups, 64 query rows each.  Per 64-key tile: S = Q K^T (wgmma, both operands in
//                    shared memory), online softmax in registers (running row maximum, the accumulator and row sum rescaled
//                    when it grows), P rounded to fp16 and fed straight from registers as the A operand of O += P V.
//   warp 8           TMA producer (one thread): Q once, then K / V^T tiles through an NS-deep mbarrier ring.
// The row sums are accumulated from the fp16-rounded P that the P V product actually uses.
// Causal mask (CLIP text encoder): key j is visible to query i only if j <= i.
//
// Replaces the baddbmm -> softmax -> bmm sequence of diffusers' CrossAttention (reached from
// riffusion/riffusion_pipeline.py:406-408) [diffusers absent: restated from memory].
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <string>

#include "rf_common.h"
#include "rf_tc.cuh"

namespace {

constexpr int TQ = 128;   // queries per CTA
constexpr int TK = 64;    // keys per tile
constexpr int ATTN_THREADS = 256 + 32;

struct AttnParams {
    int Nq, Nk, d, heads;
    int n_tiles;          // ceil(Nk / TK)
    float c;              // scale * log2(e)
    __half* out;          // [B][Nq][C]
    long out_pitch;       // C
    int causal;           // 1: key j is visible to query i only if j <= i (CLIP text encoder)
};

__device__ __forceinline__ uint32_t pack_half2(float a, float b) {
    const __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&h);
}
__device__ __forceinline__ float ex2(float a) {
    float r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(a));
    return r;
}

// DPAD: head dim rounded up to 64 (Q / K slabs of 64 elements, the tail zero-filled by TMA); NV: head dim rounded up to
// 16 (wgmma N of the P V product; V^T rows beyond d are zero-filled by TMA); NS: K / V^T ring depth
template <int DPAD, int NV, int NS>
__global__ void __launch_bounds__(ATTN_THREADS, 1)
k_flash_attn(const __grid_constant__ CUtensorMap mapQ, const __grid_constant__ CUtensorMap mapK,
             const __grid_constant__ CUtensorMap mapVt, const AttnParams p) {
    extern __shared__ __align__(1024) uint8_t smem[];
    rf_pdl_trigger();      // PDL (rf_common.h): dependents may start their prologue
    constexpr int NSLAB = DPAD / 64;
    constexpr int Q_BYTES = NSLAB * TQ * 128;
    constexpr int K_BYTES = NSLAB * TK * 128;
    constexpr int V_BYTES = ((NV * 128 + 1023) / 1024) * 1024;   // NV rows of 64 keys, padded to the swizzle atom
    uint8_t* sQ = smem;
    uint8_t* sK = sQ + Q_BYTES;                 // [NS][K_BYTES]
    uint8_t* sV = sK + NS * K_BYTES;            // [NS][V_BYTES]
    uint64_t* bars = reinterpret_cast<uint64_t*>(sV + NS * V_BYTES);
    uint64_t* q_full = bars;                    // 1
    uint64_t* kv_full = bars + 1;               // NS
    uint64_t* kv_empty = kv_full + NS;          // NS

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int q_blk = blockIdx.x, head = blockIdx.y, b = blockIdx.z;
    const int T = p.n_tiles;

    if (threadIdx.x == 0) {
        tc::mbar_init(q_full, 1);
        for (int i = 0; i < NS; ++i) {
            tc::mbar_init(&kv_full[i], 1);
            tc::mbar_init(&kv_empty[i], 256);   // every consumer thread arrives once its P V has completed
        }
        tc::fence_barrier_init();
    }
    __syncthreads();
    rf_pdl_wait();         // prologue done; the producer grid must be complete before Q / K / V are read

    if (warp == 8) {
        if (lane != 0) return;
        // ------------------------------------------------------------------ TMA producer
        tc::mbar_expect_tx(q_full, Q_BYTES);
#pragma unroll
        for (int s = 0; s < NSLAB; ++s) tc::tma_load_4d(&mapQ, q_full, sQ + s * TQ * 128, s * 64, q_blk * TQ, head, b);
        for (int j = 0; j < T; ++j) {
            const int st = j % NS;
            tc::mbar_wait(&kv_empty[st], ((j / NS) & 1) ^ 1);
            tc::mbar_expect_tx(&kv_full[st], K_BYTES + NV * 128);
#pragma unroll
            for (int s = 0; s < NSLAB; ++s)
                tc::tma_load_4d(&mapK, &kv_full[st], sK + st * K_BYTES + s * TK * 128, s * 64, j * TK, head, b);
            tc::tma_load_4d(&mapVt, &kv_full[st], sV + st * V_BYTES, j * TK, 0, head, b);
        }
        return;
    }

    // ---------------------------------------------------------------------- consumers
    const int wg = warp >> 2;
    const int frag_row = wg * 64 + (warp & 3) * 16 + (lane >> 2), frag_col = 2 * (lane & 3);
    const int q0 = q_blk * TQ + frag_row, q1 = q0 + 8;       // the two query rows of this thread
    const float c = p.c;
    float o[NV / 2];
#pragma unroll
    for (int i = 0; i < NV / 2; ++i) o[i] = 0.f;
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;   // running maxima (raw score units) and row sums
    const uint32_t q_base = tc::smem_u32(sQ) + wg * (64 * 128);
    tc::mbar_wait(q_full, 0);
    for (int j = 0; j < T; ++j) {
        const int st = j % NS;
        tc::mbar_wait(&kv_full[st], (j / NS) & 1);
        // ---- S = Q K_j^T
        float s[TK / 2];
        const uint32_t k_base = tc::smem_u32(sK + st * K_BYTES);
        tc::wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < DPAD / 16; ++kk) {
            const int sl = kk >> 2, k = kk & 3;
            tc::wgmma_ss<TK>(s, tc::make_desc_sw128(q_base + sl * TQ * 128 + k * 32),
                             tc::make_desc_sw128(k_base + sl * TK * 128 + k * 32), kk > 0 ? 1u : 0u);
        }
        tc::wgmma_commit();
        tc::wgmma_wait<0>();
        tc::reg_fence<TK / 2>(s);
        // ---- mask keys beyond Nk (zero-filled by TMA) and, causal, beyond the query index
        const int kmax0 = p.causal ? min(p.Nk, q0 + 1) : p.Nk, kmax1 = p.causal ? min(p.Nk, q1 + 1) : p.Nk;
        float mt0 = -INFINITY, mt1 = -INFINITY;
#pragma unroll
        for (int i = 0; i < TK / 8; ++i) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int key = j * TK + 8 * i + frag_col + e;
                if (key >= kmax0) s[4 * i + e] = -INFINITY;
                if (key >= kmax1) s[4 * i + 2 + e] = -INFINITY;
                mt0 = fmaxf(mt0, s[4 * i + e]);
                mt1 = fmaxf(mt1, s[4 * i + 2 + e]);
            }
        }
        mt0 = fmaxf(mt0, __shfl_xor_sync(0xffffffffu, mt0, 1));
        mt0 = fmaxf(mt0, __shfl_xor_sync(0xffffffffu, mt0, 2));
        mt1 = fmaxf(mt1, __shfl_xor_sync(0xffffffffu, mt1, 1));
        mt1 = fmaxf(mt1, __shfl_xor_sync(0xffffffffu, mt1, 2));
        const float mn0 = fmaxf(m0, mt0), mn1 = fmaxf(m1, mt1);
        // a row that has seen no visible key yet keeps maximum -inf: use 0 as its reference so that exp2 gives 0, not NaN
        const float r0 = mn0 == -INFINITY ? 0.f : mn0, r1 = mn1 == -INFINITY ? 0.f : mn1;
        const float f0 = ex2((m0 - r0) * c), f1 = ex2((m1 - r1) * c);   // 0 on the first tile (m = -inf)
        m0 = mn0;
        m1 = mn1;
        l0 *= f0;
        l1 *= f1;
#pragma unroll
        for (int i = 0; i < NV / 8; ++i) {
            o[4 * i] *= f0;
            o[4 * i + 1] *= f0;
            o[4 * i + 2] *= f1;
            o[4 * i + 3] *= f1;
        }
        // ---- P = exp2(S c - m c) in fp16, packed as the register A fragments of the P V product
        const float mc0 = r0 * c, mc1 = r1 * c;
        uint32_t pa[TK / 4];
#pragma unroll
        for (int i = 0; i < TK / 8; ++i) {
            const uint32_t h0 = pack_half2(ex2(fmaf(s[4 * i], c, -mc0)), ex2(fmaf(s[4 * i + 1], c, -mc0)));
            const uint32_t h1 = pack_half2(ex2(fmaf(s[4 * i + 2], c, -mc1)), ex2(fmaf(s[4 * i + 3], c, -mc1)));
            const float2 g0 = __half22float2(*reinterpret_cast<const __half2*>(&h0));
            const float2 g1 = __half22float2(*reinterpret_cast<const __half2*>(&h1));
            l0 += g0.x + g0.y;
            l1 += g1.x + g1.y;
            pa[2 * i] = h0;
            pa[2 * i + 1] = h1;
        }
        // ---- O += P V_j
        const uint32_t v_base = tc::smem_u32(sV + st * V_BYTES);
        tc::wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < TK / 16; ++kk)
            tc::wgmma_rs<NV>(o, pa + 4 * kk, tc::make_desc_sw128(v_base + kk * 32), 1u);
        tc::wgmma_commit();
        tc::wgmma_wait<0>();
        tc::reg_fence<NV / 2>(o);
        tc::mbar_arrive(&kv_empty[st]);
    }
    // ---- epilogue: O / rowsum -> fp16
    l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
    l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
    const float inv0 = 1.f / l0, inv1 = 1.f / l1;
    __half* dst0 = p.out + (static_cast<long>(b) * p.Nq + q0) * p.out_pitch + head * p.d;
    __half* dst1 = dst0 + 8 * p.out_pitch;
#pragma unroll
    for (int i = 0; i < NV / 8; ++i) {
        const int col = 8 * i + frag_col;
        if (col < p.d) {
            if (q0 < p.Nq) *reinterpret_cast<uint32_t*>(dst0 + col) = pack_half2(o[4 * i] * inv0, o[4 * i + 1] * inv0);
            if (q1 < p.Nq) *reinterpret_cast<uint32_t*>(dst1 + col) = pack_half2(o[4 * i + 2] * inv1, o[4 * i + 3] * inv1);
        }
    }
}

template <int DPAD, int NV, int NS>
int launch_attn(const CUtensorMap& mq, const CUtensorMap& mk, const CUtensorMap& mv, const AttnParams& p, dim3 grid,
                cudaStream_t st) {
    constexpr int NSLAB = DPAD / 64;
    constexpr int V_BYTES = ((NV * 128 + 1023) / 1024) * 1024;
    constexpr size_t smem = static_cast<size_t>(NSLAB) * TQ * 128 + static_cast<size_t>(NS) * (NSLAB * TK * 128 + V_BYTES) +
                            256 + 1024;
    static_assert(smem <= 232448, "shared memory budget (227 KB per block)");
    static rf_dev_once once;
    const cudaError_t aerr = rf_set_smem_once(once, k_flash_attn<DPAD, NV, NS>, int(smem));
    if (aerr != cudaSuccess) return rf_fail(RF_ERR_CUDA, std::string("cudaFuncSetAttribute(k_flash_attn): ") + cudaGetErrorString(aerr));
    RF_LAUNCH_PDL("k_flash_attn", (k_flash_attn<DPAD, NV, NS>), grid, dim3(ATTN_THREADS), smem, st,
                  grid.x * grid.y * grid.z <= 600u, mq, mk, mv, p);
    return RF_OK;
}

}  // namespace

// q: [B][Nq][heads*d], k: [B][Nk][heads*d], vt: [B][heads*d][vt_pitch] (V transposed), out: [B][Nq][heads*d]; fp16.
extern "C" int rf_attention_masked_f16(const void* q, const void* k, const void* vt, void* out, int B, int heads, int Nq,
                                       int Nk, int d, int vt_pitch, float scale, int causal, void* stream) {
    if (causal && (Nk > 128 || d > 112))
        return rf_fail(RF_ERR_UNSUPPORTED, "rf_attention_masked_f16: the causal mask is implemented for Nk <= 128, d <= 112 "
                                           "(the 77-token text encoder)");
    if (!q || !k || !vt || !out || B <= 0 || heads <= 0 || Nq <= 0 || Nk <= 0 || d <= 0 || (d % 8) || vt_pitch < Nk ||
        (vt_pitch % 8))
        return rf_fail(RF_ERR_INVALID, "rf_attention_masked_f16: bad argument");
    if (d > 192) return rf_fail(RF_ERR_UNSUPPORTED, "rf_attention_masked_f16: head dim > 192 (use the GEMM + softmax path)");
    const long C = static_cast<long>(heads) * d;
    const int es[4] = {1, 1, 1, 1};
    CUtensorMap mq, mk, mv;
    {
        const long dims[4] = {d, Nq, heads, B};
        const long str[4] = {1, C, d, static_cast<long>(Nq) * C};
        const int box[4] = {64, TQ, 1, 1};
        int rc = rf_tma_map_f16(&mq, q, dims, str, box, es);
        if (rc) return rc;
    }
    {
        const long dims[4] = {d, Nk, heads, B};
        const long str[4] = {1, C, d, static_cast<long>(Nk) * C};
        const int box[4] = {64, TK, 1, 1};
        int rc = rf_tma_map_f16(&mk, k, dims, str, box, es);
        if (rc) return rc;
    }
    // must equal the NV template argument of the kernel variant chosen below (the TMA box defines the bytes per stage)
    const int NV = d <= 48 ? 48 : d <= 64 ? 64 : d <= 80 ? 80 : d <= 96 ? 96 : d <= 112 ? 112 : d <= 128 ? 128 : d <= 160 ? 160 : 192;
    {
        const long dims[4] = {Nk, d, heads, B};
        const long str[4] = {1, vt_pitch, static_cast<long>(d) * vt_pitch, C * vt_pitch};
        const int box[4] = {TK, NV, 1, 1};
        int rc = rf_tma_map_f16(&mv, vt, dims, str, box, es);
        if (rc) return rc;
    }
    AttnParams p;
    p.Nq = Nq; p.Nk = Nk; p.d = d; p.heads = heads;
    p.n_tiles = (Nk + TK - 1) / TK;
    p.c = scale * 1.4426950408889634f;
    p.out = static_cast<__half*>(out);
    p.out_pitch = C;
    p.causal = causal ? 1 : 0;
    dim3 grid((Nq + TQ - 1) / TQ, heads, B);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    // ring depths: as many K / V^T stages as keep two CTAs' worth of shared memory per SM for the small head dims
    if (d <= 48) return launch_attn<64, 48, 4>(mq, mk, mv, p, grid, st);
    if (d <= 64) return launch_attn<64, 64, 4>(mq, mk, mv, p, grid, st);
    if (d <= 80) return launch_attn<128, 80, 3>(mq, mk, mv, p, grid, st);
    if (d <= 96) return launch_attn<128, 96, 3>(mq, mk, mv, p, grid, st);
    if (d <= 112) return launch_attn<128, 112, 3>(mq, mk, mv, p, grid, st);
    if (d <= 128) return launch_attn<128, 128, 3>(mq, mk, mv, p, grid, st);
    if (d <= 160) return launch_attn<192, 160, 2>(mq, mk, mv, p, grid, st);
    return launch_attn<192, 192, 2>(mq, mk, mv, p, grid, st);
}
