// Long tracks (MultiDiffusion): the window gather and the weighted overlap merge between a wide latent canvas and the
// model-sized windows the UNet runs on.  Rows are NCHW fp16; every width, stride and offset is a multiple of 8 columns,
// so both kernels move 16-byte vectors of 8 columns, and the 8 columns of a vector are covered by the same windows.
#include <cuda_fp16.h>

#include <algorithm>
#include <cstdint>

#include "rf_common.h"

static unsigned window_grid(size_t n, int threads) {
    const size_t want = (n + threads - 1) / threads;
    const size_t cap = static_cast<size_t>(rf_num_sms()) * 32;
    return static_cast<unsigned>(std::max<size_t>(1, std::min(want, cap)));
}

// in [G][C][H][Wc] -> out [G*n][C][H][Ww], out[g*n + k][c][y][x] = in[g][c][y][k*s + x]; one thread per output vector
static __global__ void k_window_gather(const uint4* __restrict__ in, int G, int CH, int Wc, int Ww, int s, int n,
                                       uint4* __restrict__ out) {
    const int Wv = Ww / 8, Wcv = Wc / 8, sv = s / 8;
    const size_t total = static_cast<size_t>(G) * n * CH * Wv;
    for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
         i += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const int xv = static_cast<int>(i % Wv);
        size_t p = i / Wv;
        const int row = static_cast<int>(p % CH);          // c * H + y
        p /= CH;
        const int k = static_cast<int>(p % n);
        const size_t g = p / n;
        out[i] = in[(g * CH + row) * Wcv + static_cast<size_t>(k) * sv + xv];
    }
}

// windows [G*n][C][H][Ww] + weights wn [n][Ww] fp32 -> canvas [G][C][H][Wc]:
// out[g][c][y][X] = fp16( sum over the windows k covering X, in increasing k, of wn[k][X - k*s] * in[g*n + k][c][y][X - k*s] )
// accumulated in fp32 and rounded once; a gather, so every output is written by one thread and no atomics are needed
static __global__ void k_window_merge(const uint4* __restrict__ in, const float* __restrict__ wn, int G, int CH, int Wc,
                                      int Ww, int s, int n, uint4* __restrict__ out) {
    const int Wv = Ww / 8, Wcv = Wc / 8;
    const size_t total = static_cast<size_t>(G) * CH * Wcv;
    for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
         i += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const int Xv = static_cast<int>(i % Wcv);
        size_t p = i / Wcv;
        const int row = static_cast<int>(p % CH);
        const size_t g = p / CH;
        const int X = Xv * 8;
        // windows k with k*s <= X < k*s + Ww
        const int k_lo = X >= Ww ? (X - Ww) / s + 1 : 0;
        const int k_hi = min(n - 1, X / s);
        float acc[8];       // from -0: a column one window covers (weight 1) is copied bit for bit, signed zeros too
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = -0.f;
        for (int k = k_lo; k <= k_hi; ++k) {
            const int x = X - k * s;
            const uint4 v = in[((g * n + k) * CH + row) * Wv + x / 8];
            const __half2* hv = reinterpret_cast<const __half2*>(&v);
            const float4 w0 = *reinterpret_cast<const float4*>(wn + static_cast<size_t>(k) * Ww + x);
            const float4 w1 = *reinterpret_cast<const float4*>(wn + static_cast<size_t>(k) * Ww + x + 4);
            const float w[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float2 f = __half22float2(hv[j]);
                acc[2 * j] = fmaf(w[2 * j], f.x, acc[2 * j]);
                acc[2 * j + 1] = fmaf(w[2 * j + 1], f.y, acc[2 * j + 1]);
            }
        }
        uint4 r;
        __half2* hr = reinterpret_cast<__half2*>(&r);
#pragma unroll
        for (int j = 0; j < 4; ++j) hr[j] = __floats2half2_rn(acc[2 * j], acc[2 * j + 1]);
        out[i] = r;
    }
}

static bool window_geometry_ok(int G, int C, int H, int Wc, int Ww, int s, int n) {
    if (G <= 0 || C <= 0 || H <= 0 || Ww <= 0 || s <= 0 || n <= 0) return false;
    if (Ww % 8 || s % 8 || Wc % 8 || s > Ww) return false;
    return static_cast<long long>(Ww) + static_cast<long long>(n - 1) * s == Wc;
}

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

extern "C" int rf_window_gather_f16(const void* canvas, int G, int C, int H, int Wc, int Ww, int s, int n, void* windows,
                                    void* stream) {
    if (!canvas || !windows || !aligned16(canvas) || !aligned16(windows) || !window_geometry_ok(G, C, H, Wc, Ww, s, n))
        return rf_fail(RF_ERR_INVALID, "rf_window_gather_f16: bad argument (Wc = Ww + (n-1) s, all multiples of 8, "
                                       "0 < s <= Ww, pointers 16-byte aligned)");
    const size_t total = static_cast<size_t>(G) * n * C * H * (Ww / 8);
    k_window_gather<<<window_grid(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const uint4*>(canvas), G, C * H, Wc, Ww, s, n, static_cast<uint4*>(windows));
    RF_CUDA_LAUNCH_CHECK("k_window_gather");
    return RF_OK;
}

extern "C" int rf_window_merge_f16(const void* windows, const float* d_weights, int G, int C, int H, int Wc, int Ww,
                                   int s, int n, void* canvas, void* stream) {
    if (!windows || !d_weights || !canvas || !aligned16(windows) || !aligned16(d_weights) || !aligned16(canvas) ||
        !window_geometry_ok(G, C, H, Wc, Ww, s, n))
        return rf_fail(RF_ERR_INVALID, "rf_window_merge_f16: bad argument (Wc = Ww + (n-1) s, all multiples of 8, "
                                       "0 < s <= Ww, pointers 16-byte aligned)");
    const size_t total = static_cast<size_t>(G) * C * H * (Wc / 8);
    k_window_merge<<<window_grid(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const uint4*>(windows), d_weights, G, C * H, Wc, Ww, s, n, static_cast<uint4*>(canvas));
    RF_CUDA_LAUNCH_CHECK("k_window_merge");
    return RF_OK;
}
