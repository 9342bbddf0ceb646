// Periodic STFT / overlap-add for seamless loops: the waveform is one period of a signal of length L = T * hop.  Frame t
// is centred at sample t * hop (torch.stft's center=True framing) and every sample index is taken modulo L, so there is no
// reflect padding and no edge: the last frames overlap the first samples.  The frame transforms are the generic engine's
// (rf_generic.cuh: k_gen_istft writes the windowed frames); only the gather and the overlap-add differ.
#pragma once
#include "rf_generic.cuh"

// STFT of frame t of clip b -> out[(b*T + t)*J + j] for the live bins; x: [B][L] one period of the signal
__global__ void __launch_bounds__(256) k_per_stft(rf_gen_tab g, const float* __restrict__ x, int L, int T,
                                                  rf_c32* __restrict__ out) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    rf_c32* A = reinterpret_cast<rf_c32*>(smem_raw);
    rf_c32* Bf = A + g.N2 + 1;
    const int t = blockIdx.x, b = blockIdx.y;
    const float* xb = x + static_cast<size_t>(b) * L;
    const int base = t * g.H - g.N / 2;                 // signal index of frame sample 0, before the modulo
    for (int n = threadIdx.x; n < g.N2; n += blockDim.x) {
        float s[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int m = 2 * n + e;
            float val = 0.f;
            if (m >= g.lo && m < g.lo + g.W) {
                int idx = (base + m) % L;
                if (idx < 0) idx += L;
                val = xb[idx] * g.window[m - g.lo];
            }
            s[e] = val;
        }
        A[n] = c_make(s[0], s[1]);
    }
    __syncthreads();
    const rf_c32* Z = rf_gen_fft<false>(A, Bf, g);
    rf_c32* dst = out + (static_cast<size_t>(b) * T + t) * g.J;
    for (int j = threadIdx.x; j < g.J; j += blockDim.x) {
        const int k = g.bins[j];
        const rf_c32 zk = Z[k == g.N2 ? 0 : k];
        const rf_c32 zc = c_conj(Z[(g.N2 - k) % g.N2]);
        const rf_c32 e = c_make(0.5f * (zk.x + zc.x), 0.5f * (zk.y + zc.y));
        const rf_c32 o = c_make(0.5f * (zk.x - zc.x), 0.5f * (zk.y - zc.y));
        const rf_c32 wo = c_mul(g.rootsN[k], o);
        dst[j] = c_make(e.x + wo.y, e.y - wo.x);
    }
}

__device__ __forceinline__ int rf_floor_div(int a, int b) { return a >= 0 ? a / b : -((-a + b - 1) / b); }

// periodic overlap-add: x[b][i] = sum of frames[t][u] over every (t, u) with t*H - c0 + u = i (mod L), divided by the sum
// of win2[u] over the same pairs.  With q = i + c0 those are the unwrapped frames t' in (q - W, q] / H, t = t' mod T,
// u = q - t' H, summed in increasing t'.  The envelope has no edge terms: for a window whose squared hop-shifted copies sum
// to a constant (Hann at W / H >= 3) it is that constant everywhere.
__global__ void k_per_ola(const float* __restrict__ frames, const float* __restrict__ win2, int T, int H, int W, int c0,
                          int L, float* __restrict__ x) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
    if (i >= L) return;
    const int q = i + c0;
    const int t_hi = rf_floor_div(q, H), t_lo = rf_floor_div(q - W, H) + 1;
    float acc = 0.f, env = 0.f;
    for (int tp = t_lo; tp <= t_hi; ++tp) {
        int t = tp % T;
        if (t < 0) t += T;
        const int u = q - tp * H;
        acc += frames[(static_cast<size_t>(b) * T + t) * W + u];
        env += win2[u];
    }
    x[static_cast<size_t>(b) * L + i] = acc / env;
}
