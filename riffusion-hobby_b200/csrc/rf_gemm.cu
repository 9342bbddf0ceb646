// Path (b) tensor-core workhorse: one wgmma / TMA kernel that computes
//     D[b][m][n] = act(alpha * sum_k A[b][m][k] * B[b][n][k] + bias) + residual          (fp16 in, fp32 accumulate)
// either as a batched "TN" GEMM (both operands K-major; linears, 1x1 convs, QK^T, PV) or as an
// implicit-GEMM 3x3 / strided convolution over NHWC activations (the im2col gather is done by the
// TMA engine: one 4-D box load per filter tap with out-of-bounds zero fill supplying the padding).
//
// CTA = one 128 x BN output tile at a time.  Warp roles: warps 0-7 = two consumer warpgroups (rows 0-63 / 64-127 of the
// tile: wgmma m64nBNk16 with both operands in shared memory), warp 8 = TMA producer (one thread), warps 9-15 = epilogue
// (the finished tile arrives through an fp32 staging tile while the consumers already run the next tile's MMAs).
// K is streamed in 64-element (128-byte, SWIZZLE_128B) slabs through a STAGES-deep mbarrier ring.
//
// Reference arithmetic this replaces (diffusers 0.9 modules reached from
// riffusion/riffusion_pipeline.py:406-408,428): torch.nn.Conv2d / Linear / baddbmm+bmm attention,
// which resolve to cuDNN / cuBLAS in the reference; none of those libraries is used here.
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <mutex>
#include <string>
#include <vector>

#include "rf_common.h"
#include "rf_tc.cuh"

namespace {

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int A_TILE_BYTES = BM * BK * 2;  // 16 KB
// two consumer warpgroups + one producer warp + seven epilogue warps.  16 warps leave each SM sub-partition (16 K
// registers, 4 of the warps) 128 registers per thread; an eighth epilogue warp would put 5 warps on one sub-partition and
// leave 96, below what the BN 160 consumers need.  Four epilogue warps were too few: the GEGLU epilogue then outlasted
// its 5-slab mainloop (DESIGN 3b).
constexpr int EPI_THREAD0 = 256 + 32;          // first epilogue thread
constexpr int EPI_THREADS = 224;
constexpr int GEMM_THREADS = EPI_THREAD0 + EPI_THREADS;
constexpr int STAGE_PAD = 4;               // fp32 staging row pitch BN + 4: row-per-thread float4 reads are conflict free

__host__ __device__ constexpr int stage_bytes(int BN) { return BM * (BN + STAGE_PAD) * 4; }

struct TcParams {
    // problem
    int M, N, K;            // GEMM mode: per-batch extents. conv mode: N = Cout, K unused
    int batch1, batch2;     // grid.z = batch1 * batch2
    int num_kb;             // K slabs
    int tiles_m, tiles_n;   // output tiles per batch entry
    int a_m1, a_m2, b_m1, b_m2;  // 0 when the operand is broadcast along that batch dimension (stride 0)
    // conv mode
    int conv;               // 0 = GEMM, 1 = conv
    int taps;               // 1 or 9
    int kc1, kc2;           // 64-channel slabs in source tensor 1 / 2 (channel concat)
    int stride, pad;        // conv stride and padding (tap (dy, dx) reads input pixel out * stride + d - pad + off)
    int tap_w;              // taps per filter row: 3 (3x3), 2 (2x2 sub-pixel phase), 1
    int off_x, off_y;       // extra tap offset (sub-pixel phases of the fused nearest-2x upsample: phase - 1 + pad)
    int osx, osy, oox, ooy; // output pixel (y, x) of the tile grid lands at (y * osy + ooy, x * osx + oox) ...
    int HoF, WoF;           // ... of an output image of HoF x WoF pixels (== Ho x Wo, scale 1, offset 0 for plain convs)
    int Ho, Wo, Bn;         // output image size and image count
    int bw, bh, bb;         // output pixels per tile: bw * bh * bb == 128
    int tiles_x, tiles_y;   // tiles per image row / column
    // epilogue
    __half* out;
    long ldo, so1, so2;     // GEMM: row pitch and batch strides of D (elements)
    const __half* bias;     // [N] (bias_mode 1) or [M] (bias_mode 2)
    int bias_mode;
    const __half* bias2;    // conv: per-image bias [Bn][bias2_pitch] (time embedding), may be null
    int bias2_pitch;
    const __half* residual; // same indexing as out, may be null
    long ldr, sr1, sr2;
    float alpha;
    int act;                // 0 none, 1 SiLU
    float* out_f32;         // optional fp32 output instead of fp16 (same indexing)
    // split-K (non-batched problems with few output tiles): work unit u = tile * splits + sp covers K slabs
    // [sp * kb_per_split, ...); every unit stores its raw fp32 accumulator to ws[sp][row][N] and k_splitk_reduce applies
    // the epilogue.  splits == 1: the normal fused epilogue.
    int splits, kb_per_split;
    float* ws;
    long ws_split_stride;   // rows * N
};

__device__ __forceinline__ float apply_act(float v, int act) {
    if (act == 1) return __fdividef(v, 1.f + __expf(-v));
    if (act == 3) return __fdividef(v, 1.f + __expf(-1.702f * v));     // quick_gelu (CLIP text encoder MLP)
    return v;
}

// exact-erf GELU  g * Phi(g),  Phi(g) = 0.5 erfc(-g / sqrt 2), branch-free with ONE MUFU op:
//   0.5 erfc(t) = 2^q(t) on t = |g| / sqrt 2 in [0, 4) (degree-7 fit of -log2 erfc(t) - 1; erfc(4) = 1.5e-8, and
//   h = 0 beyond: a clamped h = 7.7e-9 times a large negative g would give g * h, -5e-4 at g = -65504 instead of -0),
//   Phi = g < 0 ? h : 1 - h.  |error| <= 7e-7 absolute, <= 4.2e-6 relative (fp32 Horner), i.e. 1 % of an fp16 ulp —
//   same function as erff's GELU (diffusers GEGLU uses the exact form), not the tanh approximation.  erff() costs ~35
//   instructions per element on two divergent paths.
__device__ __forceinline__ float gelu_erf_fast(float g) {
    const float t = fminf(fabsf(g) * 0.70710678118654752f, 4.0f);
    float q = -2.1777638e-05f;
    q = fmaf(q, t, 0.0005068331f);
    q = fmaf(q, t, -0.005339398f);
    q = fmaf(q, t, 0.034231447f);
    q = fmaf(q, t, -0.15289085f);
    q = fmaf(q, t, -0.91675895f);
    q = fmaf(q, t, -1.6281544f);
    q = fmaf(q, t, -0.9999938f);
    float h;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(h) : "f"(q));
    return g * (g < 0.f ? (t < 4.0f ? h : 0.f) : 1.f - h);
}

// Persistent kernel: grid = min(#tiles, #SMs) CTAs, each walking work units t = blockIdx.x, +gridDim.x, ...
//   warp 8:     TMA producer — streams the K slabs of all its units through one STAGES-deep ring (phases run across units)
//   warps 0-7:  two consumer warpgroups — wgmma into register accumulators, releasing each ring stage as soon as the MMAs
//               that read it have completed; then they wait until the staging tile is free (stg_empty), write the
//               accumulators to it, arrive on stg_full and go straight on to the next unit's MMAs
//   warps 9-15: epilogue — walk the same units; per unit they wait on stg_full and run the epilogue (bias / activation /
//               residual / GEGLU / split-K partials) over the tile's 32-column row runs from the staging tile, arriving
//               on stg_empty after their last staging read.  So a tile's global stores and side-input loads overlap the
//               next tile's mainloop instead of idling the tensor pipe, which matters most where a tile has few K slabs
//               (K = 320: five).
// Tile order: n fastest, then m, then batch, so CTAs running at the same time share activation rows in L2.
//
// BRES = true (K <= BRES_KB slabs, non-batched): B-stationary.  A CTA stays on ONE column block, loads all K slabs of its
// B tile into shared memory once and streams only A through the ring while it walks the row blocks: the weight tile is
// not re-fetched from L2 for every 128-row block of the K <= 320 projections.
constexpr int BRES_KB = 5;
template <int BN, int STAGES, bool BRES = false>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
k_tc_gemm(const __grid_constant__ CUtensorMap mapA0, const __grid_constant__ CUtensorMap mapA1,
          const __grid_constant__ CUtensorMap mapB, const TcParams p) {
    extern __shared__ __align__(1024) uint8_t smem[];
    rf_pdl_trigger();      // the next kernel may start its prologue; it blocks in its own rf_pdl_wait() until this grid is done
    constexpr int B_TILE_BYTES = BN * BK * 2;
    constexpr int PITCH = BN + STAGE_PAD;
    uint8_t* sA = smem;                                      // [STAGES][A_TILE_BYTES]
    uint8_t* sB = smem + STAGES * A_TILE_BYTES;              // [STAGES][B_TILE_BYTES], BRES: [BRES_KB][B_TILE_BYTES] resident
    float* stg = reinterpret_cast<float*>(sB + (BRES ? BRES_KB : STAGES) * B_TILE_BYTES);   // [BM][PITCH]
    uint64_t* full = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(stg) + stage_bytes(BN));
    uint64_t* empty = full + STAGES;
    uint64_t* b_full = empty + STAGES;          // BRES: the resident B tile has landed
    uint64_t* stg_full = b_full + 1;            // the consumers have written a unit's accumulators to the staging tile
    uint64_t* stg_empty = stg_full + 1;         // the epilogue warps are done reading it

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tiles_mn = p.tiles_n * p.tiles_m;
    const int n_tiles = tiles_mn * p.batch1 * p.batch2 * p.splits;   // work units (== tiles when splits == 1)
    // BRES: the CTA owns column block nb_fixed and walks row blocks unit = blockIdx.x / tiles_n, + gridDim.x / tiles_n, ...
    const int nb_fixed = BRES ? static_cast<int>(blockIdx.x) % p.tiles_n : 0;
    const int unit0 = BRES ? static_cast<int>(blockIdx.x) / p.tiles_n : blockIdx.x;
    const int unit_step = BRES ? static_cast<int>(gridDim.x) / p.tiles_n : gridDim.x;
    const int n_units = BRES ? p.tiles_m : n_tiles;

    if (threadIdx.x == 0) {
        for (int i = 0; i < STAGES; ++i) {
            tc::mbar_init(&full[i], 1);
            tc::mbar_init(&empty[i], 256);      // every consumer thread arrives once it is done with the stage
        }
        tc::mbar_init(b_full, 1);
        tc::mbar_init(stg_full, 256);
        tc::mbar_init(stg_empty, EPI_THREADS);
        tc::fence_barrier_init();
    }
    if (warp == 8 && lane == 0) {
        tc::tma_prefetch_desc(&mapA0);
        tc::tma_prefetch_desc(&mapB);
    }
    __syncthreads();
    rf_pdl_wait();         // barriers and descriptors are set up: from here on global memory is touched

    if (warp == 8) {
        if (lane != 0) return;
        // ------------------------------------------------------------ TMA producer
        int it = 0;
        if constexpr (BRES) {      // the whole K extent of this CTA's B tile, once
            tc::mbar_expect_tx(b_full, p.num_kb * B_TILE_BYTES);
            for (int kb = 0; kb < p.num_kb; ++kb)
                tc::tma_load_4d(&mapB, b_full, sB + kb * B_TILE_BYTES, kb * BK, nb_fixed * BN, 0, 0);
        }
        for (int unit = unit0; unit < n_units; unit += unit_step) {
            const int tile = BRES ? unit * p.tiles_n + nb_fixed : unit / p.splits, sp = BRES ? 0 : unit - (unit / p.splits) * p.splits;
            const int kb0 = sp * p.kb_per_split, kb1 = min(p.num_kb, kb0 + p.kb_per_split);
            const int z = tile / tiles_mn, mn = tile - z * tiles_mn;
            const int m_blk = mn / p.tiles_n, n_blk = mn - m_blk * p.tiles_n;
            const int b1 = z % p.batch1, b2 = z / p.batch1;
            int tx = 0, ty = 0, tb = 0;
            if (p.conv) {
                tx = m_blk % p.tiles_x;
                ty = (m_blk / p.tiles_x) % p.tiles_y;
                tb = m_blk / (p.tiles_x * p.tiles_y);
            }
            for (int kb = kb0; kb < kb1; ++kb, ++it) {
                const int stage = it % STAGES;
                const uint32_t phase = (it / STAGES) & 1;
                tc::mbar_wait(&empty[stage], phase ^ 1);
                tc::mbar_expect_tx(&full[stage], A_TILE_BYTES + (BRES ? 0 : B_TILE_BYTES));
                void* dstA = sA + stage * A_TILE_BYTES;
                void* dstB = sB + stage * B_TILE_BYTES;
                if (!p.conv) {
                    tc::tma_load_4d(&mapA0, &full[stage], dstA, kb * BK, m_blk * BM, b1 * p.a_m1, b2 * p.a_m2);
                    if (!BRES) tc::tma_load_4d(&mapB, &full[stage], dstB, kb * BK, n_blk * BN, b1 * p.b_m1, b2 * p.b_m2);
                } else {
                    const int kct = p.kc1 + p.kc2;
                    const int tap = kb / kct, kc = kb - tap * kct;
                    const int dy = tap / p.tap_w, dx = tap - dy * p.tap_w;
                    const int x0 = tx * p.bw * p.stride + dx - p.pad + p.off_x;
                    const int y0 = ty * p.bh * p.stride + dy - p.pad + p.off_y;
                    if (kc < p.kc1)
                        tc::tma_load_4d(&mapA0, &full[stage], dstA, kc * BK, x0, y0, tb * p.bb);
                    else
                        tc::tma_load_4d(&mapA1, &full[stage], dstA, (kc - p.kc1) * BK, x0, y0, tb * p.bb);
                    if (!BRES) tc::tma_load_4d(&mapB, &full[stage], dstB, kb * BK, n_blk * BN, 0, 0);
                }
            }
        }
        return;
    }

    if (warp < 8) {
        // ------------------------------------------------------------ consumers (threads 0-255)
        const int wg = warp >> 2;                    // rows [64 wg, +64) of the tile
        const int frag_row = wg * 64 + (warp & 3) * 16 + (lane >> 2), frag_col = 2 * (lane & 3);
        if constexpr (BRES) tc::mbar_wait(b_full, 0);
        int it = 0, done = 0;                        // units done: the staging tile's phase
        for (int unit = unit0; unit < n_units; unit += unit_step, ++done) {
            const int sp = BRES ? 0 : unit - (unit / p.splits) * p.splits;
            const int kb0 = sp * p.kb_per_split, kb1 = min(p.num_kb, kb0 + p.kb_per_split);
            // ---- main loop: one wgmma group per stage, at most one group in flight behind the newest
            float acc[BN / 2];
#pragma unroll
            for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
            int prev = -1;
            for (int kb = kb0; kb < kb1; ++kb, ++it) {
                const int stage = it % STAGES;
                tc::mbar_wait(&full[stage], (it / STAGES) & 1);
                const uint32_t a_base = tc::smem_u32(sA + stage * A_TILE_BYTES) + wg * (64 * 128);
                const uint32_t b_base = tc::smem_u32(sB + (BRES ? kb : stage) * B_TILE_BYTES);
                tc::wgmma_fence();
#pragma unroll
                for (int k = 0; k < BK / 16; ++k)
                    tc::wgmma_ss<BN>(acc, tc::make_desc_sw128(a_base + k * 32), tc::make_desc_sw128(b_base + k * 32), 1u);
                tc::wgmma_commit();
                tc::wgmma_wait<1>();                 // the group of the previous stage has completed: release that stage
                tc::reg_fence<BN / 2>(acc);
                if (prev >= 0) tc::mbar_arrive(&empty[prev]);
                prev = stage;
            }
            tc::wgmma_wait<0>();
            tc::reg_fence<BN / 2>(acc);
            if (prev >= 0) tc::mbar_arrive(&empty[prev]);

            // ---- accumulators -> fp32 staging tile, once the epilogue warps are done with the previous unit's
            tc::mbar_wait(stg_empty, (done & 1) ^ 1);
#pragma unroll
            for (int i = 0; i < BN / 8; ++i) {
                const int c = 8 * i + frag_col;
                *reinterpret_cast<float2*>(stg + frag_row * PITCH + c) = make_float2(acc[4 * i], acc[4 * i + 1]);
                *reinterpret_cast<float2*>(stg + (frag_row + 8) * PITCH + c) = make_float2(acc[4 * i + 2], acc[4 * i + 3]);
            }
            tc::mbar_arrive(stg_full);
        }
        return;
    }

    // ---------------------------------------------------------------- epilogue (threads 288-511)
    constexpr int RUNS = BM * (BN / 32);         // 32-column runs of one row each: run r = row r % BM, columns 32 (r / BM) ...
    // 64 bytes (one 32-column run of fp16 side input) as four 128-bit loads
    auto ld64 = [](const __half* src, uint4* q4) {
        const uint4* s4 = reinterpret_cast<const uint4*>(src);
#pragma unroll
        for (int j = 0; j < 4; ++j) q4[j] = s4[j];
    };
    int done = 0;
    for (int unit = unit0; unit < n_units; unit += unit_step, ++done) {
        const int tile = BRES ? unit * p.tiles_n + nb_fixed : unit / p.splits, sp = BRES ? 0 : unit - (unit / p.splits) * p.splits;
        const int z = tile / tiles_mn, mn = tile - z * tiles_mn;
        const int m_blk = mn / p.tiles_n, n_blk = mn - m_blk * p.tiles_n;
        const int b1 = z % p.batch1, b2 = z / p.batch1;
        int tx = 0, ty = 0, tb = 0;
        if (p.conv) {
            tx = m_blk % p.tiles_x;
            ty = (m_blk / p.tiles_x) % p.tiles_y;
            tb = m_blk / (p.tiles_x * p.tiles_y);
        }
        tc::mbar_wait(stg_full, done & 1);
        // thread t takes the runs t, t + EPI_THREADS, ...: a warp reads 32 consecutive rows of one column range
#pragma unroll 1
        for (int r = threadIdx.x - EPI_THREAD0; r < RUNS; r += EPI_THREADS) {
            const int row = r % BM, c0 = (r / BM) * 32;
            float f[32];
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const float4 t = *reinterpret_cast<const float4*>(stg + row * PITCH + c0 + 4 * i);
                f[4 * i] = t.x; f[4 * i + 1] = t.y; f[4 * i + 2] = t.z; f[4 * i + 3] = t.w;
            }
            if (r + EPI_THREADS >= RUNS) tc::mbar_arrive(stg_empty);   // this thread's last staging read of the unit
            bool row_ok;
            long out_off, res_off;
            int img = 0;
            if (!p.conv) {
                const int m = m_blk * BM + row;
                row_ok = m < p.M;
                out_off = static_cast<long>(b2) * p.so2 + static_cast<long>(b1) * p.so1 + static_cast<long>(m) * p.ldo;
                res_off = static_cast<long>(b2) * p.sr2 + static_cast<long>(b1) * p.sr1 + static_cast<long>(m) * p.ldr;
            } else {
                const int xi = row % p.bw, yi = (row / p.bw) % p.bh, bi = row / (p.bw * p.bh);
                const int x = tx * p.bw + xi, y = ty * p.bh + yi;
                img = tb * p.bb + bi;
                row_ok = (x < p.Wo) && (y < p.Ho) && (img < p.Bn);
                const long pix = (static_cast<long>(img) * p.HoF + (y * p.osy + p.ooy)) * p.WoF + (x * p.osx + p.oox);
                out_off = pix * p.ldo;
                res_off = pix * p.ldr;
            }
            const int n0 = n_blk * BN + c0;
            if (!row_ok || n0 >= p.N) continue;
            const float bias_row = p.bias_mode == 2 ? __half2float(p.bias[m_blk * BM + row]) : 0.f;
            if (p.splits > 1) {   // raw partial sums; ws rows are dense with pitch N in output-row order
                float* wp = p.ws + sp * p.ws_split_stride + (out_off / p.ldo) * p.N + n0;
                if (n0 + 32 <= p.N && (p.N & 3) == 0) {
#pragma unroll
                    for (int i = 0; i < 8; ++i)
                        reinterpret_cast<float4*>(wp)[i] = make_float4(f[4 * i], f[4 * i + 1], f[4 * i + 2], f[4 * i + 3]);
                } else {
                    for (int i = 0; i < 32; ++i)
                        if (n0 + i < p.N) wp[i] = f[i];
                }
                continue;
            }
#pragma unroll
            for (int i = 0; i < 32; ++i) f[i] = f[i] * p.alpha + bias_row;
            const bool full_run = n0 + 32 <= p.N;
            // per-column bias and per-image bias: 16-byte loads when the 32-column run is complete and aligned
            if (p.bias_mode == 1) {
                if (full_run && ((reinterpret_cast<uintptr_t>(p.bias + n0) & 15) == 0)) {
                    uint4 q4[4];
                    ld64(p.bias + n0, q4);
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const uint4 bv = q4[j];
                        const __half2* bh = reinterpret_cast<const __half2*>(&bv);
#pragma unroll
                        for (int e = 0; e < 4; ++e) {
                            const float2 t = __half22float2(bh[e]);
                            f[8 * j + 2 * e] += t.x;
                            f[8 * j + 2 * e + 1] += t.y;
                        }
                    }
                } else {
                    for (int i = 0; i < 32; ++i)
                        if (n0 + i < p.N) f[i] += __half2float(p.bias[n0 + i]);
                }
            }
            if (p.bias2) {
                const __half* b2p = p.bias2 + static_cast<long>(img) * p.bias2_pitch + n0;
                if (full_run && ((reinterpret_cast<uintptr_t>(b2p) & 15) == 0)) {
                    uint4 q4[4];
                    ld64(b2p, q4);
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const uint4 bv = q4[j];
                        const __half2* bh = reinterpret_cast<const __half2*>(&bv);
#pragma unroll
                        for (int e = 0; e < 4; ++e) {
                            const float2 t = __half22float2(bh[e]);
                            f[8 * j + 2 * e] += t.x;
                            f[8 * j + 2 * e + 1] += t.y;
                        }
                    }
                } else {
                    for (int i = 0; i < 32; ++i)
                        if (n0 + i < p.N) f[i] += __half2float(b2p[i]);
                }
            }
            if (p.act == 2) {
                // GEGLU: the 32-column run is [16 value | 16 gate] columns of the same 16 outputs (weight rows
                // interleaved by the caller); D has N/2 columns: out[n0/2 + j] = value_j * gelu(gate_j)
                __half* dst = p.out + out_off + (n0 >> 1);
                uint32_t pk[8];
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const float g0 = f[16 + 2 * j], g1 = f[17 + 2 * j];
                    const float y0 = f[2 * j] * gelu_erf_fast(g0);
                    const float y1 = f[2 * j + 1] * gelu_erf_fast(g1);
                    const __half2 h = __floats2half2_rn(y0, y1);
                    pk[j] = *reinterpret_cast<const uint32_t*>(&h);
                }
                reinterpret_cast<uint4*>(dst)[0] = make_uint4(pk[0], pk[1], pk[2], pk[3]);
                reinterpret_cast<uint4*>(dst)[1] = make_uint4(pk[4], pk[5], pk[6], pk[7]);
                continue;
            }
            if (p.act) {
#pragma unroll
                for (int i = 0; i < 32; ++i) f[i] = apply_act(f[i], p.act);
            }
            if (p.residual) {
                const __half* rp = p.residual + res_off + n0;
                if (full_run && ((reinterpret_cast<uintptr_t>(rp) & 15) == 0)) {
                    uint4 q4[4];
                    ld64(rp, q4);
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const uint4 rv = q4[j];
                        const __half2* rh = reinterpret_cast<const __half2*>(&rv);
#pragma unroll
                        for (int e = 0; e < 4; ++e) {
                            const float2 t = __half22float2(rh[e]);
                            f[8 * j + 2 * e] += t.x;
                            f[8 * j + 2 * e + 1] += t.y;
                        }
                    }
                } else {
                    for (int i = 0; i < 32; ++i)
                        if (n0 + i < p.N) f[i] += __half2float(rp[i]);
                }
            }
            if (p.out_f32) {
                for (int i = 0; i < 32; ++i)
                    if (n0 + i < p.N) p.out_f32[out_off + n0 + i] = f[i];
            } else if (full_run && ((reinterpret_cast<uintptr_t>(p.out + out_off + n0) & 15) == 0)) {
                uint4* dst = reinterpret_cast<uint4*>(p.out + out_off + n0);
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    __half2 h0 = __floats2half2_rn(f[8 * i + 0], f[8 * i + 1]);
                    __half2 h1 = __floats2half2_rn(f[8 * i + 2], f[8 * i + 3]);
                    __half2 h2 = __floats2half2_rn(f[8 * i + 4], f[8 * i + 5]);
                    __half2 h3 = __floats2half2_rn(f[8 * i + 6], f[8 * i + 7]);
                    dst[i] = make_uint4(*reinterpret_cast<uint32_t*>(&h0), *reinterpret_cast<uint32_t*>(&h1),
                                        *reinterpret_cast<uint32_t*>(&h2), *reinterpret_cast<uint32_t*>(&h3));
                }
            } else {
                for (int i = 0; i < 32; ++i)
                    if (n0 + i < p.N) p.out[out_off + n0 + i] = __float2half_rn(f[i]);
            }
        }
    }
}

// ------------------------------------------------------------------------------ host side
// optional live measurement (bench.py): CUDA events around every tensor-core launch + algorithmic FLOP count
struct TcProfile {
    bool on = false;
    std::vector<cudaEvent_t> ev;   // begin/end pairs
    double flops = 0.0;
    long launches = 0;
    struct Rec { int conv, M, N, K, batch, splits, bn; };   // bn < 0: CTA-pair kernel
    std::vector<Rec> recs;
};

TcProfile g_prof;
std::mutex g_prof_mu;

template <int BN, int STAGES, bool BRES = false>
int launch(const CUtensorMap& a0, const CUtensorMap& a1, const CUtensorMap& b, const TcParams& p, dim3 grid,
           cudaStream_t st) {   // `grid` arrives as (tiles_n, tiles_m, batch) and is flattened to a persistent 1-D grid
    constexpr size_t smem = static_cast<size_t>(STAGES) * A_TILE_BYTES +
                            static_cast<size_t>(BRES ? BRES_KB : STAGES) * (BN * BK * 2) + stage_bytes(BN) + 1024;
    static_assert(smem <= 232448, "shared memory budget (227 KB per block)");
    const int num_sms = rf_num_sms();
    const int n_tiles = static_cast<int>(grid.x * grid.y * grid.z);
    if (BRES) {   // every CTA is bound to one column block: a multiple of tiles_n CTAs
        grid = dim3(static_cast<unsigned>((num_sms / p.tiles_n) * p.tiles_n));
    } else {
        grid = dim3(static_cast<unsigned>(n_tiles < num_sms ? n_tiles : num_sms));
    }
    static rf_dev_once once;
    const cudaError_t aerr = rf_set_smem_once(once, k_tc_gemm<BN, STAGES, BRES>, int(smem));
    if (aerr != cudaSuccess) return rf_fail(RF_ERR_CUDA, std::string("cudaFuncSetAttribute: ") + cudaGetErrorString(aerr));
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    const bool prof = g_prof.on;
    if (prof) {
        RF_CUDA_TRY(cudaEventCreate(&e0));
        RF_CUDA_TRY(cudaEventCreate(&e1));
        RF_CUDA_TRY(cudaEventRecord(e0, st));
    }
    RF_LAUNCH_PDL("k_tc_gemm", (k_tc_gemm<BN, STAGES, BRES>), grid, dim3(GEMM_THREADS), smem, st, n_tiles <= 2 * num_sms,
                  a0, a1, b, p);
    if (prof) {
        RF_CUDA_TRY(cudaEventRecord(e1, st));
        std::lock_guard<std::mutex> lk(g_prof_mu);
        g_prof.ev.push_back(e0);
        g_prof.ev.push_back(e1);
        g_prof.launches += 1;
        const double m = p.conv ? static_cast<double>(p.Bn) * p.Ho * p.Wo : static_cast<double>(p.M) * p.batch1 * p.batch2;
        g_prof.flops += 2.0 * m * p.N * p.K;
        g_prof.recs.push_back({p.conv, p.conv ? p.Bn * p.Ho * p.Wo : p.M, p.N, p.K, p.batch1 * p.batch2, p.splits,
                               BRES ? 1000 + BN : BN});
    }
    return RF_OK;
}

// ---- split-K second stage: out = act(alpha * sum_s ws[s] + bias + bias2[img]) + residual, 8 columns per thread
__global__ void k_splitk_reduce(const float* __restrict__ ws, int splits, long split_stride, long rows, int N, long ldo,
                                long ldr, int rows_per_image, float alpha, const __half* __restrict__ bias, int bias_mode,
                                const __half* __restrict__ bias2, int bias2_pitch, int act,
                                const __half* __restrict__ residual, __half* __restrict__ out, float* __restrict__ out_f32) {
    const int n8 = N / 8;
    for (long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x; i < rows * n8;
         i += static_cast<long>(gridDim.x) * blockDim.x) {
        const long r = i / n8;
        const int n0 = static_cast<int>(i - r * n8) * 8;
        float f[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) f[e] = 0.f;
        for (int sidx = 0; sidx < splits; ++sidx) {
            const float4* wp = reinterpret_cast<const float4*>(ws + sidx * split_stride + r * N + n0);
            const float4 a = wp[0], b = wp[1];
            f[0] += a.x; f[1] += a.y; f[2] += a.z; f[3] += a.w;
            f[4] += b.x; f[5] += b.y; f[6] += b.z; f[7] += b.w;
        }
        const float brow = bias_mode == 2 ? __half2float(bias[r]) : 0.f;
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            float v = f[e] * alpha + brow;
            if (bias_mode == 1) v += __half2float(bias[n0 + e]);
            if (bias2) v += __half2float(bias2[(r / rows_per_image) * bias2_pitch + n0 + e]);
            if (act == 1 || act == 3) v = apply_act(v, act);
            if (residual) v += __half2float(residual[r * ldr + n0 + e]);
            f[e] = v;
        }
        if (out_f32) {
#pragma unroll
            for (int e = 0; e < 8; ++e) out_f32[r * ldo + n0 + e] = f[e];
        } else {
            uint32_t pk[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const __half2 h = __floats2half2_rn(f[2 * e], f[2 * e + 1]);
                pk[e] = *reinterpret_cast<const uint32_t*>(&h);
            }
            *reinterpret_cast<uint4*>(out + r * ldo + n0) = make_uint4(pk[0], pk[1], pk[2], pk[3]);
        }
    }
}

// Split-K workspace: caller-provided scratch (desc.workspace / workspace_bytes, sized by rf_*_workspace_bytes) — the
// library keeps no mutable state, so concurrent calls on different streams are safe.  Without it split-K is not used.
constexpr size_t SPLIT_WS_MAX = static_cast<size_t>(192) << 20;

// Number of K splits: a problem with fewer tiles than SMs leaves SMs idle AND streams its weights through too few
// TMA rings to cover HBM latency.  Cost model in microseconds: ceil(units / SMs) waves of (slabs per unit) x t_slab,
// plus for S > 1 the second-stage launch and its fp32 round trip (mostly L2 resident).
int pick_splits(long rows, int N, int tiles, int num_kb, int num_sms, bool allowed) {
    static const char* env = getenv("RF_GEMM_SPLITK");   // "0" disables, "N" forces N where legal (A/B measurements)
    if (!allowed || (env && env[0] == '0')) return 1;
    const double t_slab = 0.2, t_launch = 3.0, ws_bw = 8.0e6;   // us, us, bytes/us
    int best = 1;
    double best_t = 1e30;
    for (int S = 1; S <= 8; ++S) {
        if (S > 1 && (num_kb / S < 6 || static_cast<size_t>(S) * rows * N * 4 > SPLIT_WS_MAX)) break;
        const int kbs = (num_kb + S - 1) / S;
        if (S > 1 && (S - 1) * kbs >= num_kb) continue;   // the last split would be empty
        const int waves = (tiles * S + num_sms - 1) / num_sms;
        double t = waves * kbs * t_slab;
        if (S > 1) t += t_launch + 2.0 * S * rows * N * 4 / ws_bw;
        if (env && atoi(env) == S) return S;
        if (t < best_t * (S > 1 ? 0.9 : 1.0)) {   // a split must win by 10%
            best_t = t;
            best = S;
        }
    }
    return best;
}

// Output-tile width: 64 for narrow outputs; otherwise 128, or 160 when it divides N and is not slower by the wave
// count: relative time = ceil(tiles / SMs) waves x tile width.  160 always wins when 128 does not divide N (N = 320:
// two exact tiles instead of three with 17 % padding) and often when both do; it also moves 12 % fewer operand bytes
// per FLOP from L2.  RF_GEMM_BN=<64|128|160> forces a width where it is legal (A/B measurements, parity tests).
int pick_bn(int N, long tiles_m) {
    if (const char* env = getenv("RF_GEMM_BN")) {        // read per call: the parity tests flip it inside one process
        const int bn = atoi(env);
        if (bn == 64 || bn == 128 || (bn == 160 && N % 160 == 0)) return bn;
    }
    if (N <= 64) return 64;
    if (N % 160) return 128;
    const long sms = rf_num_sms();
    const long t128 = tiles_m * ((N + 127) / 128), t160 = tiles_m * (N / 160);
    const long c128 = ((t128 + sms - 1) / sms) * 128, c160 = ((t160 + sms - 1) / sms) * 160;
    return c160 * 100 <= c128 * 102 ? 160 : 128;
}

int dispatch(int N, int bn, const CUtensorMap& a0, const CUtensorMap& a1, const CUtensorMap& b, TcParams& p,
             int tiles_m, int nbatch, cudaStream_t st, void* ws, size_t ws_bytes, size_t* query) {
    // one persistent CTA per SM: TMA ring of 4-6 stages of one 64-wide K slab each.  BN 160 takes 4, which fills the 227 KB
    // next to the staging tile exactly: with 3 the deep-K convs waited on operand latency (DESIGN 3b, "Ring depth")
    p.tiles_n = (N + bn - 1) / bn;
    p.tiles_m = tiles_m;
    // split-K: non-batched, plain or SiLU epilogue, 16-byte aligned fp16/fp32 rows
    const long rows = p.conv ? static_cast<long>(p.Bn) * p.Ho * p.Wo : p.M;
    const bool can_split = nbatch == 1 && p.act != 2 && (N % 8) == 0 && (p.ldo % 8) == 0 && (!p.conv || p.osx == 1) &&
                           (!p.residual || (p.ldr % 8) == 0) &&
                           ((reinterpret_cast<uintptr_t>(p.out ? static_cast<void*>(p.out) : static_cast<void*>(p.out_f32)) & 15) == 0);
    p.splits = pick_splits(rows, N, p.tiles_n * tiles_m, p.num_kb, rf_num_sms(), can_split);
    p.kb_per_split = (p.num_kb + p.splits - 1) / p.splits;
    p.ws = nullptr;
    p.ws_split_stride = rows * N;
    if (p.splits > 1) {
        const size_t need = static_cast<size_t>(p.splits) * rows * N * sizeof(float);
        if (query) {
            *query = need;
            return RF_OK;
        }
        if (!ws || ws_bytes < need) {          // no (or too small a) workspace: the un-split kernel is always correct
            p.splits = 1;
            p.kb_per_split = p.num_kb;
        } else {
            p.ws = static_cast<float*>(ws);
        }
    }
    if (query) {
        *query = 0;
        return RF_OK;
    }
    dim3 grid(p.tiles_n * p.splits, tiles_m, nbatch);
    int rc;
    const char* env_bres = getenv("RF_GEMM_BRES");
    if (bn == 160 && nbatch == 1 && p.splits == 1 && p.num_kb <= BRES_KB && p.tiles_n <= 8 &&
        static_cast<long>(tiles_m) * p.tiles_n >= 4L * rf_num_sms() && !(env_bres && env_bres[0] == '0')) {
        return launch<160, 2, true>(a0, a1, b, p, grid, st);       // B-stationary (K <= 320, N = 160 k)
    }
    if (bn == 160) rc = launch<160, 4>(a0, a1, b, p, grid, st);   // N = 320-type layers: two exact 160-column tiles
    else if (bn == 128) rc = launch<128, 4>(a0, a1, b, p, grid, st);
    else rc = launch<64, 6>(a0, a1, b, p, grid, st);
    if (rc || p.splits == 1) return rc;
    const long work = rows * (N / 8);
    const unsigned blocks = static_cast<unsigned>(std::min<long>((work + 255) / 256, 8L * rf_num_sms()));
    k_splitk_reduce<<<blocks, 256, 0, st>>>(p.ws, p.splits, p.ws_split_stride, rows, N, p.ldo, p.ldr,
                                            p.conv ? p.Ho * p.Wo : 1, p.alpha, p.bias, p.bias_mode, p.bias2, p.bias2_pitch,
                                            p.act, p.residual, p.out, p.out_f32);
    RF_CUDA_LAUNCH_CHECK("k_splitk_reduce");
    if (g_prof.on) {   // the measured interval of this launch ends after the second stage
        std::lock_guard<std::mutex> lk(g_prof_mu);
        if (!g_prof.ev.empty()) RF_CUDA_TRY(cudaEventRecord(g_prof.ev.back(), st));
    }
    return RF_OK;
}

}  // namespace

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
    static PFN_encodeTiled fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* sym = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &sym, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<PFN_encodeTiled>(sym);
    });
    return fn;
}

int rf_tma_map_f16(CUtensorMap* map, const void* ptr, const long dims[4], const long strides[4], const int box[4],
                   const int estrides[4]) {
    PFN_encodeTiled enc = get_encode();
    if (!enc) return rf_fail(RF_ERR_CUDA, "cuTensorMapEncodeTiled unavailable (no CUDA driver)");
    cuuint64_t gdim[4], gstr[3];
    cuuint32_t bx[4], es[4];
    for (int i = 0; i < 4; ++i) {
        gdim[i] = static_cast<cuuint64_t>(dims[i]);
        bx[i] = static_cast<cuuint32_t>(box[i]);
        es[i] = static_cast<cuuint32_t>(estrides[i]);
        if (i) {
            gstr[i - 1] = static_cast<cuuint64_t>(strides[i]) * 2;
            if (gstr[i - 1] % 16) return rf_fail(RF_ERR_INVALID, "tensor map: stride not a multiple of 16 bytes");
        }
    }
    if (reinterpret_cast<uintptr_t>(ptr) % 16) return rf_fail(RF_ERR_INVALID, "tensor map: base not 16-byte aligned");
    CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(ptr), gdim, gstr, bx, es,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return rf_fail(RF_ERR_CUDA, "cuTensorMapEncodeTiled failed: " + std::to_string(int(r)));
    return RF_OK;
}

// ------------------------------------------------------------------------------ C-ABI
static int gemm_impl(const rf_gemm_desc* d, void* stream, size_t* query) {
    if (!d || !d->A || !d->B || !d->D || d->M <= 0 || d->N <= 0 || d->K <= 0)
        return rf_fail(RF_ERR_INVALID, "rf_gemm_f16: bad argument");
    const int b1 = d->batch1 > 0 ? d->batch1 : 1, b2 = d->batch2 > 0 ? d->batch2 : 1;
    // a batch stride of 0 means "broadcast": the map gets extent 1 there and the kernel passes coordinate 0
    const int a_m1 = (b1 > 1 && d->sa1 != 0) ? 1 : 0, a_m2 = (b2 > 1 && d->sa2 != 0) ? 1 : 0;
    const int b_m1 = (b1 > 1 && d->sb1 != 0) ? 1 : 0, b_m2 = (b2 > 1 && d->sb2 != 0) ? 1 : 0;
    CUtensorMap ma, mb;
    {
        const long dims[4] = {d->K, d->M, a_m1 ? b1 : 1, a_m2 ? b2 : 1};
        const long str[4] = {1, d->lda, a_m1 ? d->sa1 : d->lda, a_m2 ? d->sa2 : d->lda};
        const int box[4] = {BK, BM, 1, 1};
        const int es[4] = {1, 1, 1, 1};
        int rc = rf_tma_map_f16(&ma, d->A, dims, str, box, es);
        if (rc) return rc;
    }
    const int bn = pick_bn(d->N, static_cast<long>((d->M + BM - 1) / BM) * b1 * b2);
    {
        const long dims[4] = {d->K, d->N, b_m1 ? b1 : 1, b_m2 ? b2 : 1};
        const long str[4] = {1, d->ldb, b_m1 ? d->sb1 : d->ldb, b_m2 ? d->sb2 : d->ldb};
        const int box[4] = {BK, bn, 1, 1};
        const int es[4] = {1, 1, 1, 1};
        int rc = rf_tma_map_f16(&mb, d->B, dims, str, box, es);
        if (rc) return rc;
    }
    TcParams p{};
    p.M = d->M; p.N = d->N; p.K = d->K;
    p.batch1 = b1; p.batch2 = b2;
    p.num_kb = (d->K + BK - 1) / BK;
    p.conv = 0;
    p.a_m1 = a_m1; p.a_m2 = a_m2; p.b_m1 = b_m1; p.b_m2 = b_m2;
    p.out = static_cast<__half*>(d->out_f32 ? nullptr : d->D);
    p.out_f32 = static_cast<float*>(d->out_f32 ? d->D : nullptr);
    p.ldo = d->ldd; p.so1 = d->sd1; p.so2 = d->sd2;
    p.bias = static_cast<const __half*>(d->bias);
    p.bias_mode = d->bias ? d->bias_mode : 0;
    p.bias2 = nullptr;
    p.residual = static_cast<const __half*>(d->residual);
    p.ldr = d->ldr; p.sr1 = d->sr1; p.sr2 = d->sr2;
    p.alpha = d->alpha == 0.f ? 1.f : d->alpha;
    p.act = d->act;
    if (d->act == 2 && ((d->N % 32) || d->residual || d->out_f32 || (d->ldd % 8) || (d->sd1 % 8) || (d->sd2 % 8) ||
                        (reinterpret_cast<uintptr_t>(d->D) & 15)))
        return rf_fail(RF_ERR_UNSUPPORTED, "rf_gemm_f16: GEGLU epilogue needs N % 32 == 0, fp16 output with 16-byte "
                                           "aligned rows and no residual");
    return dispatch(d->N, bn, ma, ma, mb, p, (d->M + BM - 1) / BM, b1 * b2, static_cast<cudaStream_t>(stream), d->workspace,
                    d->workspace_bytes > 0 ? static_cast<size_t>(d->workspace_bytes) : 0, query);
}

extern "C" int rf_gemm_f16(const rf_gemm_desc* d, void* stream) { return gemm_impl(d, stream, nullptr); }
extern "C" size_t rf_gemm_workspace_bytes(const rf_gemm_desc* d) {
    size_t need = 0;
    return gemm_impl(d, nullptr, &need) == RF_OK ? need : 0;
}

static int conv_impl(const rf_conv_desc* d, void* stream, size_t* query) {
    if (!d || !d->x1 || !d->w || !d->out || d->B <= 0 || d->H <= 0 || d->W <= 0 || d->C1 <= 0 || d->Cout <= 0)
        return rf_fail(RF_ERR_INVALID, "rf_conv2d_f16: bad argument");
    if (d->pad_mode < 0 || d->pad_mode > 4) return rf_fail(RF_ERR_INVALID, "rf_conv2d_f16: pad_mode must be 0 to 4");
    const bool up2 = d->pad_mode == 2 || d->pad_mode == 4;   // nearest-2x upsample fused in: four 2x2 sub-pixel convolutions
    const int halo = d->pad_mode >= 3 ? 1 : 0;  // x1 carries its one-pixel border (rf_pad_wrap_w_f16): read it, pad nothing
    if (up2 && (d->ksize != 2 || d->stride != 1 || d->x2 || d->residual))
        return rf_fail(RF_ERR_UNSUPPORTED, "rf_conv2d_f16: pad_mode 2 / 4 (fused upsample) takes ksize 2 phase weights, "
                                           "stride 1, one input, no residual");
    if (halo && (d->x2 || (!up2 && d->ksize != 3) || d->H < 3 || d->W < 3))
        return rf_fail(RF_ERR_UNSUPPORTED, "rf_conv2d_f16: pad_mode 3 / 4 (input with a one-pixel border) takes a 3x3 or "
                                           "fused-upsample convolution of one input of at least 3x3 pixels");
    if (!up2 && d->ksize != 1 && d->ksize != 3) return rf_fail(RF_ERR_UNSUPPORTED, "rf_conv2d_f16: kernel size must be 1 or 3");
    if (d->stride != 1 && d->stride != 2) return rf_fail(RF_ERR_UNSUPPORTED, "rf_conv2d_f16: stride must be 1 or 2");
    if ((d->C1 % BK) || (d->x2 && (d->C2 % BK)))
        return rf_fail(RF_ERR_UNSUPPORTED, "rf_conv2d_f16: channel counts must be multiples of 64 (use the direct "
                                           "convolution for the 4- and 3-channel layers)");
    const int pad = (d->ksize == 3 && d->pad_mode == 0) ? 1 : 0;
    const int extra = (d->ksize == 3 && d->pad_mode == 1) ? 1 : 0;   // one implicit zero row/column at the far edge
    // up2: the tile grid is the input grid (without its border); pad_mode 3 is a 3x3 convolution with padding 0
    const int Ho = up2 ? d->H - 2 * halo : (d->H + 2 * pad + extra - d->ksize) / d->stride + 1;
    const int Wo = up2 ? d->W - 2 * halo : (d->W + 2 * pad + extra - d->ksize) / d->stride + 1;
    // output pixels per tile.  bw is a power of two (it must divide 128): among those from min(8, bw_max) up to bw_max,
    // the largest power of two <= min(Wo, 128), take the one that pads Wo least, the larger one on a tie.  Powers of two
    // keep bw = Wo; 96-, 48- and 24-wide levels (768-pixel-wide clips) get exact 32-, 16- and 8-wide tiles instead of
    // padding a quarter of the columns.
    int bw_max = Wo >= 128 ? 128 : Wo;
    while (BM % bw_max) --bw_max;
    int bw = bw_max;
    for (int c = bw_max / 2; c >= 8; c /= 2)
        if ((Wo + c - 1) / c * c < (Wo + bw - 1) / bw * bw) bw = c;
    int bh = BM / bw;
    if (bh > Ho) bh = Ho;
    while ((BM / bw) % bh) --bh;
    const int bb = BM / (bw * bh);
    const int C2 = d->x2 ? d->C2 : 0;
    CUtensorMap m1, m2, mb;
    const int s = d->stride;
    {
        const long dims[4] = {d->C1, d->W, d->H, d->B};
        const long str[4] = {1, d->C1, static_cast<long>(d->W) * d->C1, static_cast<long>(d->H) * d->W * d->C1};
        const int box[4] = {BK, (bw - 1) * s + 1, (bh - 1) * s + 1, bb};
        const int es[4] = {1, s, s, 1};
        int rc = rf_tma_map_f16(&m1, d->x1, dims, str, box, es);
        if (rc) return rc;
    }
    m2 = m1;
    if (d->x2) {
        const long dims[4] = {C2, d->W, d->H, d->B};
        const long str[4] = {1, C2, static_cast<long>(d->W) * C2, static_cast<long>(d->H) * d->W * C2};
        const int box[4] = {BK, (bw - 1) * s + 1, (bh - 1) * s + 1, bb};
        const int es[4] = {1, s, s, 1};
        int rc = rf_tma_map_f16(&m2, d->x2, dims, str, box, es);
        if (rc) return rc;
    }
    const int taps = d->ksize * d->ksize;
    const long Ktot = static_cast<long>(taps) * (d->C1 + C2);
    const long conv_tiles_m = static_cast<long>((Wo + bw - 1) / bw) * ((Ho + bh - 1) / bh) * ((d->B + bb - 1) / bb);
    const int bn = pick_bn(d->Cout, conv_tiles_m);
    {
        const long dims[4] = {Ktot, d->Cout, 1, 1};
        const long str[4] = {1, Ktot, Ktot * d->Cout, Ktot * d->Cout};
        const int box[4] = {BK, bn, 1, 1};
        const int es[4] = {1, 1, 1, 1};
        int rc = rf_tma_map_f16(&mb, d->w, dims, str, box, es);
        if (rc) return rc;
    }
    TcParams p{};
    p.M = 0; p.N = d->Cout; p.K = static_cast<int>(Ktot);
    p.batch1 = 1; p.batch2 = 1;
    p.conv = 1; p.taps = taps;
    p.kc1 = d->C1 / BK; p.kc2 = C2 / BK;
    p.num_kb = taps * (p.kc1 + p.kc2);
    p.stride = s; p.pad = pad;
    p.tap_w = d->ksize; p.off_x = 0; p.off_y = 0;
    p.osx = 1; p.osy = 1; p.oox = 0; p.ooy = 0;
    p.Ho = Ho; p.Wo = Wo; p.Bn = d->B;
    p.HoF = Ho; p.WoF = Wo;
    p.bw = bw; p.bh = bh; p.bb = bb;
    p.tiles_x = (Wo + bw - 1) / bw;
    p.tiles_y = (Ho + bh - 1) / bh;
    const int tiles_b = (d->B + bb - 1) / bb;
    p.out = static_cast<__half*>(d->out);
    p.out_f32 = nullptr;
    p.ldo = d->Cout; p.ldr = d->Cout;
    p.bias = static_cast<const __half*>(d->bias);
    p.bias_mode = d->bias ? 1 : 0;
    p.bias2 = static_cast<const __half*>(d->bias_per_image);
    p.bias2_pitch = d->bias_per_image_pitch > 0 ? d->bias_per_image_pitch : d->Cout;
    p.residual = static_cast<const __half*>(d->residual);
    p.alpha = d->alpha == 0.f ? 1.f : d->alpha;
    p.act = d->act;
    void* ws = d->workspace;
    const size_t ws_bytes = d->workspace_bytes > 0 ? static_cast<size_t>(d->workspace_bytes) : 0;
    if (!up2) return dispatch(d->Cout, bn, m1, m2, mb, p, p.tiles_x * p.tiles_y * tiles_b, 1, static_cast<cudaStream_t>(stream), ws,
                              ws_bytes, query);
    // conv3x3(pad 1) of the nearest-2x upsampled image == four 2x2 convolutions of the input, one per output parity
    // (py, px): output (2y + py, 2x + px) reads input rows y + py - 1 + {0, 1} and columns x + px - 1 + {0, 1}; the 3x3 taps
    // that fall on the same input pixel are pre-summed in the phase weights w[phase][Cout][2][2][Cin] (9 -> 4 taps: 2.25x
    // fewer FLOPs, and the upsampled tensor is never written).
    p.osx = 2; p.osy = 2; p.HoF = 2 * Ho; p.WoF = 2 * Wo;
    for (int ph = 0; ph < 4; ++ph) {
        const int py = ph >> 1, px = ph & 1;
        p.off_y = py - 1 + halo; p.off_x = px - 1 + halo;
        p.ooy = py; p.oox = px;
        CUtensorMap mph;
        const long dims[4] = {Ktot, d->Cout, 1, 1};
        const long str[4] = {1, Ktot, Ktot * d->Cout, Ktot * d->Cout};
        const int box[4] = {BK, bn, 1, 1};
        const int es[4] = {1, 1, 1, 1};
        int rc = rf_tma_map_f16(&mph, static_cast<const __half*>(d->w) + static_cast<long>(ph) * d->Cout * Ktot, dims, str, box, es);
        if (rc) return rc;
        TcParams q = p;
        rc = dispatch(d->Cout, bn, m1, m2, mph, q, p.tiles_x * p.tiles_y * tiles_b, 1, static_cast<cudaStream_t>(stream), nullptr, 0,
                      query);      // strided outputs: never split
        if (rc || query) return rc;
    }
    return RF_OK;
}

extern "C" int rf_conv2d_f16(const rf_conv_desc* d, void* stream) { return conv_impl(d, stream, nullptr); }
extern "C" size_t rf_conv2d_workspace_bytes(const rf_conv_desc* d) {
    size_t need = 0;
    return conv_impl(d, nullptr, &need) == RF_OK ? need : 0;
}

// Live measurement aid for bench.py: between begin and end every rf_gemm_f16 / rf_conv2d_f16 launch is bracketed
// by CUDA events on its stream and its algorithmic FLOPs (2*M*N*K with the true, un-padded extents) are summed.
extern "C" int rf_tc_profile_begin(void) {
    std::lock_guard<std::mutex> lk(g_prof_mu);
    g_prof.on = true;
    g_prof.flops = 0.0;
    g_prof.launches = 0;
    g_prof.recs.clear();
    for (cudaEvent_t e : g_prof.ev) cudaEventDestroy(e);
    g_prof.ev.clear();
    return RF_OK;
}
extern "C" int rf_tc_profile_end(double* ms_out, double* flops_out, long* launches_out) {
    std::lock_guard<std::mutex> lk(g_prof_mu);
    g_prof.on = false;
    double ms = 0.0;
    cudaError_t err = cudaDeviceSynchronize();
    FILE* dump = nullptr;
    if (const char* path = getenv("RF_TC_PROFILE_DUMP")) dump = fopen(path, "w");   // per-launch csv (A/B measurements)
    if (dump) fprintf(dump, "conv,M,N,K,batch,splits,bn,ms\n");
    for (size_t i = 0; i + 1 < g_prof.ev.size() && err == cudaSuccess; i += 2) {
        float t = 0.f;
        err = cudaEventElapsedTime(&t, g_prof.ev[i], g_prof.ev[i + 1]);
        ms += t;
        if (dump && i / 2 < g_prof.recs.size()) {
            const TcProfile::Rec& r = g_prof.recs[i / 2];
            fprintf(dump, "%d,%d,%d,%d,%d,%d,%d,%.4f\n", r.conv, r.M, r.N, r.K, r.batch, r.splits, r.bn, t);
        }
    }
    if (dump) fclose(dump);
    for (cudaEvent_t e : g_prof.ev) cudaEventDestroy(e);
    g_prof.ev.clear();
    if (ms_out) *ms_out = ms;
    if (flops_out) *flops_out = g_prof.flops;
    if (launches_out) *launches_out = g_prof.launches;
    if (err != cudaSuccess) return rf_fail(RF_ERR_CUDA, std::string("rf_tc_profile_end: ") + cudaGetErrorString(err));
    return RF_OK;
}
