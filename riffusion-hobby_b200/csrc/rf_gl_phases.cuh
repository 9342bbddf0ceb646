// Phase functions of the STFT / iSTFT kernels.  Every phase is a function of (tid, nthreads)
// with no intra-phase cross-thread dependency, so the CUDA kernels call them with
// __syncthreads() in between and tests/hostemu runs them as plain loops over tid (a
// CPU emulation of the device control flow — test infrastructure only).
//
// Algorithm (see DESIGN.md §3): two consecutive frames (t, t+1) are packed as the real and
// imaginary part of one complex sequence z[n'] over the 4410 live samples of the
// 17640-sample frame.  Bin k = 4m + r of the 17640-point DFT is the m-th output of a
// 4410-point DFT of z[n'] * exp(-2 pi i r n'/17640); the 4410-point DFT is a twiddle-free
// prime-factor 10 x 9 x 49 three-dimensional DFT held in shared memory as V[a][b][c]
// (position a*441 + b*49 + c).  One CTA handles one "group" (r in {0,2} or r in {1,3}) so
// that a bin and its Hermitian partner N-k live in the same CTA.
//
// Pass order and thread mapping are chosen for few shared-memory bank conflicts:
//   forward: radix-9 over b fused with gather/window/modulate (items (a, c) in the plan's annealed slot order,
//            rf_pass_b_perm.inc) -> radix-10 / radix-5 over a (lanes over consecutive positions) -> radix-49 over c as two
//            7-thread phases (lane stride 49 = 1 mod 16 eight-byte banks)
//   inverse: radix-49 -> radix-10 / 5 -> radix-9 fused with demodulate/window/overlap-add.
#pragma once
#include <math.h>
#include <stddef.h>
#include <stdint.h>

#include "rf_dft.cuh"

#define RF_PW 4410
#define RF_PN 17640
#define RF_NT 256                              // threads per CTA of the FFT kernels
#define RF_LOAD_UNROLL 4

// The passes are templated on NA, the size of the "a" axis of the prime-factor grid:
//   NA = 10: full-rate transform, W = 4410 samples per frame (n' = 441a + 490b + 90c mod 4410)
//   NA = 5 : time-decimated transform used inside the Griffin-Lim loop when the live band allows it:
//            only every second sample of the waveform is carried (W = 2205, n'' = 441a + 245b + 45c mod 2205),
//            the bins k = 4m + r of the 17640-grid become outputs of 2205-point DFTs (period 8820 in k).
// Shared-memory position of (a, b, c) is a*441 + b*49 + c in both cases.
template <int NA> struct rf_geom {
    static constexpr int W = NA * 441;          // complex points per sub-transform
    static constexpr int SB = W / 9;            // index step of b in the time-side (Ruritanian) map
    static constexpr int SC = W / 49;           // index step of c
    static constexpr int B_ITEMS = 49 * NA;     // (a, c) items of the fused radix-9 pass
    static constexpr int B_ITERS = (B_ITEMS + RF_NT - 1) / RF_NT;
};

struct alignas(16) rf_f4 {
    float x, y, z, w;
};

// Tables of one prime-factor grid (rf_bin_tabs in rf_plan.h holds the host copies and the exact definitions)
struct rf_gl_tables {
    const rf_f4* wg_fwd;   // [9][49 NA] per (b, item): (w0, w1, cos t, -sin t): windows of frames t0 / t0+1 (sample parities for
                           // NA = 5) and the modulation exp(-i t) of r = 1 at that sample; r = 2, 3 are derived from it
    const rf_f4* wg_inv;   // same layout: (w0/N, w1/N, cos t, sin t)
    const uint32_t* items; // [49 NA] radix-9 pass item of slot tau: V position a*441 + c | first sample index n'(a, b=0, c) << 12
    const uint32_t* bt;    // [n_live] V offset of the bin | V offset of its Hermitian partner << 14 | self-paired << 31
    const rf_f4* ab_inv;   // [n_live] (alpha, beta):  Z[k] = alpha C0 + beta C1,  Z[N-k] = conj(alpha C0 - beta C1)
    const rf_f4* ab_fwd;   // [n_live] (gamma, delta): X_t[k] = gamma (Z[k] + conj Z[N-k]),  X_t+1[k] = delta (Z[k] - conj Z[N-k])
    const uint16_t* zpos;  // V offsets that no bin of the group writes: nz0 entries of group 0, then nz1 of group 1
    const float* zero_row; // [n_live] zeros: the magnitudes of a frame that does not exist (odd frame count)
    int nz0, nz1;
    int n_live;
    int n_even;
    int off1;              // offset of frame t0+1 in the staged sample buffer: hop (NA = 10) or (hop+1)/2 (NA = 5)
};

// streaming (evict-first) loads for the spectra, which are read once per launch: the per-bin tables stay in L1
#ifndef RF_GL_LD_CG
#define RF_GL_LD_CG 0      // 1: ld.global.cg (L2 only) instead of ld.global.cs (evict-first) — A/B builds
#endif
#if defined(__CUDA_ARCH__)
RF_HD float rf_ld_stream(const float* p) { return RF_GL_LD_CG ? __ldcg(p) : __ldcs(p); }
RF_HD rf_c32 rf_ld_stream(const rf_c32* p) {
    const float2 v = RF_GL_LD_CG ? __ldcg(reinterpret_cast<const float2*>(p)) : __ldcs(reinterpret_cast<const float2*>(p));
    return c_make(v.x, v.y);
}
#else
RF_HD float rf_ld_stream(const float* p) { return *p; }
RF_HD rf_c32 rf_ld_stream(const rf_c32* p) { return *p; }
#endif

// ------------------------------------------------------------------ shared passes
// radix-10 over a: items (s, b, c); lanes run over consecutive positions
template <bool INV, int NA>
RF_HD void rf_pass_a(int tid, int nt, rf_c32* V) {
    constexpr int W = rf_geom<NA>::W;
    for (int it = tid; it < 2 * 441; it += nt) {
        const int s = it / 441;
        rf_c32* p = V + s * W + (it - s * 441);
        rf_c32 v[NA];
#pragma unroll
        for (int a = 0; a < NA; ++a) v[a] = p[441 * a];
        if (NA == 10) dft10<INV>(v);
        else dft5<INV>(v[0], v[1], v[2], v[3], v[4]);
#pragma unroll
        for (int a = 0; a < NA; ++a) p[441 * a] = v[a];
    }
}

// radix-49 over c, SEVEN threads per 49-point transform (work item w = j * transforms + transform), two phases with a barrier
// in between, both in place and free of cross-thread hazards:
//   column phase (thread j = c2): DFT7 over the stride-7 elements p[7 c1 + j], twiddle w49^(k1 j), back to p[7 k1 + j]
//   row phase    (thread j = k1): DFT7 over the contiguous row p[7 j + c2], back to p[7 j + k2] = X[j + 7 k2]
// forward = column phase then row phase: natural time order in, TRANSPOSED spectral order out (X[k] at 7 (k % 7) + k / 7,
// which is what the plan's position tables pp / pp2 point at: rf_pfa_spec_pos);  inverse = row phase (twiddle after the
// DFT) then column phase: transposed spectral order in, natural time order out.  One thread per transform (the previous
// form) kept 49 complex values = 98 registers live and left 166 of 256 threads idle for NA = 5.
#ifndef RF_GL_PASS7
#define RF_GL_PASS7 1       // 0: the one-thread-per-transform radix-49 pass (A/B builds)
#endif
template <bool INV, int NA, int STEP>
RF_HD void rf_pass_c7(int tid, int nt, rf_c32* V) {
#if !RF_GL_PASS7
    if (STEP == 0) {
        for (int it = tid; it < 2 * 9 * NA; it += nt) {
            rf_c32* p = V + it * 49;
            rf_c32 v[49];
#pragma unroll
            for (int c = 0; c < 49; ++c) v[c] = p[c];
            dft49<INV>(v);
#pragma unroll
            for (int c = 0; c < 49; ++c) p[c] = v[7 * (c % 7) + c / 7];
        }
    }
    return;
#endif
    const float sg = INV ? 1.0f : -1.0f;
    constexpr bool COLUMN = (STEP == 0) != INV;
    constexpr int NTR = 2 * 9 * NA;         // 49-point transforms in V
    for (int w = tid; w < NTR * 7; w += nt) {
        // lanes run over the transforms (stride 49 elements = 1 mod 16 eight-byte banks: conflict-free in both phases) and
        // j is uniform over (most of) a warp, so the twiddle reads below are constant-cache broadcasts
        const int j = w / NTR, it = w - j * NTR;
        rf_c32* p = V + it * 49;  // s*W + ab*49 == it*49
        rf_c32 v[7];
        if (COLUMN) {
#pragma unroll
            for (int i = 0; i < 7; ++i) v[i] = p[7 * i + j];
        } else {
#pragma unroll
            for (int i = 0; i < 7; ++i) v[i] = p[7 * j + i];
        }
        dft7<INV>(v[0], v[1], v[2], v[3], v[4], v[5], v[6]);
        if (STEP == 0) {   // the twiddle sits between the two DFT7 stages: after the first phase in either direction
#pragma unroll
            for (int i = 1; i < 7; ++i) v[i] = c_mulk(v[i], rf_w49_cos(i * j), sg * rf_w49_sin(i * j));
        }
        if (COLUMN) {
#pragma unroll
            for (int i = 0; i < 7; ++i) p[7 * i + j] = v[i];
        } else {
#pragma unroll
            for (int i = 0; i < 7; ++i) p[7 * j + i] = v[i];
        }
    }
}

// ------------------------------------------------------------------ forward (STFT)
// xs[0 .. W+hop): padded signal starting at the first live sample of frame t0; frame t0+1 is
// xs[hop + n'].  First pass: gather, window*modulate (two r values), radix-9 over b.
template <int NA>
RF_HD void rf_stft_pass_b(int tid, int nt, rf_c32* V, const float* xs, const rf_gl_tables& tb, int g,
                          bool has1) {
    constexpr int W = rf_geom<NA>::W, SB = rf_geom<NA>::SB;
    // sub-transform r of the group sees z[n'] exp(-2 pi i r n'/N):  r0 = g, r1 = g + 2, so with y = (x0 w0) + i (x1 w1) and
    // c = exp(-i t):  u0 = y c^g,  u1 = u0 c^2.  Items (a, c) are assigned to slots tau by the plan (bank-conflict-free order).
    for (int tau = tid; tau < rf_geom<NA>::B_ITEMS; tau += nt) {
        const uint32_t item = tb.items[tau];
        const int base = item >> 12;
        rf_c32 u0[9], u1[9];
#pragma unroll
        for (int b = 0; b < 9; ++b) {
            int n = base + SB * b;
            if (n >= W) n -= W;
            const float x0 = xs[n], x1 = has1 ? xs[tb.off1 + n] : 0.f;
            const rf_f4 f = tb.wg_fwd[b * (49 * NA) + tau];
            rf_c32 y = c_make(x0 * f.x, x1 * f.y);
            const rf_c32 c1 = c_make(f.z, f.w);
            const rf_c32 c2 = c_make(f.z * f.z - f.w * f.w, 2.f * f.z * f.w);
            if (g) y = c_mul(y, c1);
            u0[b] = y;
            u1[b] = c_mul(y, c2);
        }
        dft9<false>(u0);
        dft9<false>(u1);
        rf_c32* p = V + (item & 4095u);
#pragma unroll
        for (int b = 0; b < 9; ++b) {
            p[49 * b] = u0[b];
            p[W + 49 * b] = u1[b];
        }
    }
}

// Unpack the pair: X_t[k] and X_{t+1}[k] for the live bins j in [j0, j1) of this group.
// out0/out1: rows of the [T][n_live] spectrum for frames t0, t0+1 (out1 may be null).
//   X_t[k]   = ph (Z[k] + conj Z[N-k]) / 2 = gamma u,   X_t+1[k] = ph po (Z[k] - conj Z[N-k]) / 2i = delta v
// (ph = exp(-2 pi i 3k/8): frame offset; po = exp(-2 pi i k/N): the odd-sample frame of a decimated pair)
template <int NA, bool F1, int U, bool TAIL>
RF_HD void rf_stft_post_batch(int jb, int j1, int nt, const rf_c32* V, const rf_gl_tables& tb, rf_c32* out0, rf_c32* out1) {
    const uint32_t* pbt = tb.bt + jb;
    const rf_f4* pgd = tb.ab_fwd + jb;
    rf_c32* o0 = out0 + jb;
    rf_c32* o1 = F1 ? out1 + jb : nullptr;
    uint32_t pw[U];
    rf_f4 gd[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
        const int o = TAIL ? ((jb + u * nt < j1) ? u * nt : 0) : u * nt;
        pw[u] = pbt[o];
        gd[u] = pgd[o];
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
        if (TAIL && u > 0 && jb + u * nt >= j1) continue;
        const rf_c32 zk = V[pw[u] & 16383u];
        const rf_c32 zp = V[(pw[u] >> 14) & 16383u];
        o0[u * nt] = c_mul(c_make(gd[u].x, gd[u].y), c_make(zk.x + zp.x, zk.y - zp.y));
        if (F1) o1[u * nt] = c_mul(c_make(gd[u].z, gd[u].w), c_make(zk.x - zp.x, zk.y + zp.y));
    }
}
template <int NA, bool F1>
RF_HD void rf_stft_post_t(int tid, int nt, const rf_c32* V, const rf_gl_tables& tb, int j0, int j1, rf_c32* out0,
                          rf_c32* out1) {
    int jb = j0 + tid;
    for (; jb + 3 * nt < j1; jb += 4 * nt) rf_stft_post_batch<NA, F1, 4, false>(jb, j1, nt, V, tb, out0, out1);
    if (jb < j1) rf_stft_post_batch<NA, F1, 4, true>(jb, j1, nt, V, tb, out0, out1);
}
template <int NA>
RF_HD void rf_stft_post(int tid, int nt, const rf_c32* V, const rf_gl_tables& tb, int j0, int j1, rf_c32* out0,
                        rf_c32* out1) {
    if (out1) rf_stft_post_t<NA, true>(tid, nt, V, tb, j0, j1, out0, out1);
    else rf_stft_post_t<NA, false>(tid, nt, V, tb, j0, j1, out0, out1);
}

// ------------------------------------------------------------------ inverse (iSTFT)
// NA = 10: clear V (a barrier must follow).  NA = 5: the live bins and their partners cover all but a few hundred of the
// 4410 slots, so only the uncovered slots (zpos) are cleared — disjoint from what rf_istft_load writes: no barrier in between.
template <int NA>
RF_HD void rf_istft_zero(int tid, int nt, rf_c32* V, const rf_gl_tables& tb, int g) {
    if (NA == 5) {
        const uint16_t* z = tb.zpos + (g ? tb.nz0 : 0);
        const int n = g ? tb.nz1 : tb.nz0;
        for (int i = tid; i < n; i += nt) V[z[i]] = c_make(0.f, 0.f);
    } else {
        for (int i = tid; i < 2 * rf_geom<NA>::W; i += nt) V[i] = c_make(0.f, 0.f);
    }
}

// Griffin-Lim phase update fused into the load:
//   mode 0: coefficient = S * A0            (A0 = cur: the caller's initial angles)
//   mode 1: A = R - m*Rprev ; A /= (|A| + 1e-16) ; coefficient = S * A
//           (TA/functional/functional.py:337-340; no momentum term on the first update)
// The normalisation is one reciprocal square root (MUFU.RSQ, ~1 ulp) instead of sqrt + two IEEE divisions: torch's
// own complex abs() is a hypot with a rounding of its own, so neither form is bit-identical to the reference, and a
// 1-ulp change of a unit phasor is the same size as the rounding differences between any two FFT implementations.
// |A| < 1e-15 (a bin with no energy) is clamped instead of adding 1e-16: the product with S is noise either way.
template <int MODE, bool UP>
RF_HD rf_c32 rf_gl_coef(float S, rf_c32 a, rf_c32 q, float momentum) {
    if (MODE) {
        if (UP) {
            a.x = fmaf(-momentum, q.x, a.x);
            a.y = fmaf(-momentum, q.y, a.y);
        }
        const float n2 = fmaxf(fmaf(a.x, a.x, a.y * a.y), 1e-30f);
#if defined(__CUDA_ARCH__)
        float rs;   // n2 >= 1e-30 is a normal number: the flush-to-zero form needs no denormal pre-scaling
        asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(rs) : "f"(n2));
        S *= rs;
#else
        S *= 1.0f / sqrtf(n2);
#endif
    }
    return c_make(S * a.x, S * a.y);
}

struct rf_istft_in {
    const float* S0;      // magnitudes, frame t0   [n_live]
    const float* S1;      // frame t0+1; a chunk that ends on a single frame passes tb.zero_row here (and frame t0's cur / prev rows)
    const rf_c32* cur0;   // R (or A0) rows
    const rf_c32* cur1;
    const rf_c32* prev0;  // previous R rows or null
    const rf_c32* prev1;
    int mode;
    float momentum;
};

// Coefficients of the packed pair, per live bin k of the group (C0, C1 = the two frames' Griffin-Lim coefficients):
//   Z[k] = conj(ph) (C0 + i C1') = alpha C0 + beta C1,   Z[N-k] = ph (conj C0 + i conj C1') = conj(alpha C0 - beta C1)
// with C1' = C1 conj(po); alpha, beta are per-bin constants (rf_bin_tabs), so the phase factors cost two complex products.
// All global loads of a batch of RF_LOAD_UNROLL bins are issued before any is used, so one DRAM latency is paid per
// batch instead of per bin.  MODE / UP (update mode, momentum term present) are uniform over a launch and compiled out.
// TAIL: the last batch of a thread, slots past j1 are dropped (their loads are clamped onto the last bin, not predicated:
// every thread then makes the same number of load -> use round trips, which is what the phase waits on)
template <int NA, int MODE, bool UP, int U, bool TAIL>
RF_HD void rf_istft_load_batch(int jb, int j1, int nt, rf_c32* V, const rf_gl_tables& tb, const rf_istft_in& in) {
    // bins jb, jb + nt, ..: one base pointer per array, the slots are constant offsets from it
    const uint32_t* pbt = tb.bt + jb;
    const rf_f4* pab = tb.ab_inv + jb;
    const float* pS0 = in.S0 + jb;
    const rf_c32* pA0 = in.cur0 + jb;
    const rf_c32* pQ0 = UP ? in.prev0 + jb : nullptr;
    const float* pS1 = in.S1 + jb;
    const rf_c32* pA1 = in.cur1 + jb;
    const rf_c32* pQ1 = UP ? in.prev1 + jb : nullptr;
    const float mom = in.momentum;
    uint32_t pw[U];
    rf_f4 ab[U];
    float s0[U], s1[U];
    rf_c32 a0[U], a1[U], q0[U], q1[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
        const int o = TAIL ? ((jb + u * nt < j1) ? u * nt : 0) : u * nt;
        pw[u] = pbt[o];
        ab[u] = pab[o];
        s0[u] = rf_ld_stream(pS0 + o);
        a0[u] = rf_ld_stream(pA0 + o);
        if (UP) q0[u] = rf_ld_stream(pQ0 + o);
        s1[u] = rf_ld_stream(pS1 + o);
        a1[u] = rf_ld_stream(pA1 + o);
        if (UP) q1[u] = rf_ld_stream(pQ1 + o);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
        if (TAIL && u > 0 && jb + u * nt >= j1) continue;
        const uint32_t p = pw[u];
        const rf_c32 c0 = rf_gl_coef<MODE, UP>(s0[u], a0[u], UP ? q0[u] : c_make(0.f, 0.f), mom);
        const rf_c32 c1 = rf_gl_coef<MODE, UP>(s1[u], a1[u], UP ? q1[u] : c_make(0.f, 0.f), mom);
        const rf_c32 al = c_make(ab[u].x, ab[u].y), be = c_make(ab[u].z, ab[u].w);
        rf_c32* vk = V + (p & 16383u);
        if (static_cast<int32_t>(p) < 0) {   // self-paired bin (DC / Nyquist, rarely live): irfft ignores the imaginary part
            const rf_c32 P = c_mul(al, c_make(c0.x, 0.f)), Q = c_mul(be, c_make(c1.x, 0.f));
            *vk = c_make(P.x + Q.x, P.y + Q.y);
            continue;
        }
        const rf_c32 P = c_mul(al, c0);
        const rf_c32 Q = c_mul(be, c1);
        rf_c32* vp = V + ((p >> 14) & 16383u);
        *vk = c_make(P.x + Q.x, P.y + Q.y);
        *vp = c_make(P.x - Q.x, Q.y - P.y);
    }
}

template <int NA, int MODE, bool UP>
RF_HD void rf_istft_load_t(int tid, int nt, rf_c32* V, const rf_gl_tables& tb, int j0, int j1, const rf_istft_in& in) {
    int jb = j0 + tid;
    for (; jb + 3 * nt < j1; jb += 4 * nt) rf_istft_load_batch<NA, MODE, UP, 4, false>(jb, j1, nt, V, tb, in);
    if (jb < j1) rf_istft_load_batch<NA, MODE, UP, 4, true>(jb, j1, nt, V, tb, in);
}

template <int NA>
RF_HD void rf_istft_load(int tid, int nt, rf_c32* V, const rf_gl_tables& tb, int j0, int j1, const rf_istft_in& in) {
    if (in.mode == 0) rf_istft_load_t<NA, 0, false>(tid, nt, V, tb, j0, j1, in);
    else if (in.prev0 != nullptr) rf_istft_load_t<NA, 1, true>(tid, nt, V, tb, j0, j1, in);
    else rf_istft_load_t<NA, 1, false>(tid, nt, V, tb, j0, j1, in);
}

// Last inverse pass: radix-9 over b for both sub-FFTs, demodulate, window (x 1/N), overlap-add.
// ola points at the chunk accumulator position of frame t0's first live sample; frame t0+1
// lands hop samples later.  The add of frame t0+1 at n'+hop aliases the add of frame t0 at
// n'' = n'+hop done by ANOTHER thread, so the real-part adds and the imaginary-part adds are
// separated by a barrier:
//   which = 0: real-part adds only, 1: imaginary-part adds only (the host emulation runs the
//   function twice), 2: both with __syncthreads() in between (device).
// Every thread executes the same number of iterations so the barrier is convergent.
template <int NA>
RF_HD void rf_istft_pass_b(int tid, int nt, const rf_c32* V, float* ola, const rf_gl_tables& tb, int g,
                           bool has1, int which) {
    constexpr int W = rf_geom<NA>::W, SB = rf_geom<NA>::SB;
    constexpr int ITERS = rf_geom<NA>::B_ITERS;
    float re[ITERS][9], im[ITERS][9];
    int base_n[ITERS];
#pragma unroll
    for (int itn = 0; itn < ITERS; ++itn) {
        const int tau = tid + itn * nt;
        if (tau < rf_geom<NA>::B_ITEMS) {
            const uint32_t item = tb.items[tau];
            base_n[itn] = item >> 12;
            const rf_c32* p = V + (item & 4095u);
            rf_c32 u0[9], u1[9];
#pragma unroll
            for (int b = 0; b < 9; ++b) {
                u0[b] = p[49 * b];
                u1[b] = p[W + 49 * b];
            }
            dft9<true>(u0);
            dft9<true>(u1);
#pragma unroll
            for (int b = 0; b < 9; ++b) {
                // z = (w/N) e^g (u0 + u1 e^2), e = exp(+i t): frame t0 = w0 Re z, frame t0+1 = w1 Im z
                const rf_f4 f = tb.wg_inv[b * (49 * NA) + tau];
                const rf_c32 e1 = c_make(f.z, f.w);
                const rf_c32 e2 = c_make(f.z * f.z - f.w * f.w, 2.f * f.z * f.w);
                rf_c32 t = c_add(u0[b], c_mul(u1[b], e2));
                if (g) t = c_mul(t, e1);
                re[itn][b] = f.x * t.x;
                im[itn][b] = f.y * t.y;
            }
        }
    }
    if (which != 1) {
#pragma unroll
        for (int itn = 0; itn < ITERS; ++itn)
            if (tid + itn * nt < rf_geom<NA>::B_ITEMS) {
#pragma unroll
                for (int b = 0; b < 9; ++b) {
                    int n = base_n[itn] + SB * b;
                    if (n >= W) n -= W;
                    ola[n] += re[itn][b];
                }
            }
    }
#if defined(__CUDA_ARCH__)
    if (which == 2) __syncthreads();
#endif
    if (which != 0 && has1) {
#pragma unroll
        for (int itn = 0; itn < ITERS; ++itn)
            if (tid + itn * nt < rf_geom<NA>::B_ITEMS) {
#pragma unroll
                for (int b = 0; b < 9; ++b) {
                    int n = base_n[itn] + SB * b;
                    if (n >= W) n -= W;
                    ola[tb.off1 + n] += im[itn][b];
                }
            }
    }
}

// ------------------------------------------------------------------ staging / assembly
RF_HD int rf_reflect_index(int i, int L) {
    if (i < 0) i = -i;
    else if (i >= L) i = 2 * (L - 1) - i;
    return i;
}

// xs[i] = x_padded[t0*hop + i] for i in [0, W+hop), with torch.stft's reflect padding
// (center=True, pad_mode="reflect") applied on the fly to the un-padded signal x[0..L).
// x points at waveform sample `base` (base = 0 for a whole waveform; the decimated loop keeps only the two full-rate
// edge strips [0, E) and [L-E, L), see rf_gl_dec_geom)
RF_HD void rf_stage_x(int tid, int nt, float* xs, const float* x, int L, int t0, int hop, int base = 0) {
    const int q0 = t0 * hop - RF_PW / 2;
    for (int i = tid; i < RF_PW + hop; i += nt) {
        const int ii = rf_reflect_index(q0 + i, L);
        xs[i] = (ii >= 0 && ii < L) ? x[ii - base] : 0.f;
    }
}

// window envelope of torch.istft at sample i of the kept region: sum of w^2 of covering frames
RF_HD float rf_envelope(int i, const float* win2, int T, int H, int W) {
    const int q = W / 2 + i;  // hop coordinates: frame t covers [tH, tH+W)
    const int t_hi = (T - 1 < q / H) ? T - 1 : q / H;
    int t_lo = (q - W + H) / H;  // ceil((q-W+1)/H)
    if (q - W + 1 <= 0) t_lo = 0;
    float env = 0.f;
    for (int t = t_lo; t <= t_hi; ++t) env += win2[q - t * H];
    return env;
}

// One output sample of torch.istft's overlap-add: sum of the chunk partial sums that cover
// sample i of the kept region, divided by the window envelope.  part: [2 groups][nchunks][PL]
RF_HD float rf_ola_sample(int i, const float* part, float env, int T, int G, int PL, int nchunks,
                          int H, int W) {
    const int q = W / 2 + i;
    const int t_hi = (T - 1 < q / H) ? T - 1 : q / H;
    int t_lo = (q - W + H) / H;
    if (q - W + 1 <= 0) t_lo = 0;
    const int c_lo = t_lo / G, c_hi = t_hi / G;
    float acc = 0.f;
    for (int g = 0; g < 2; ++g)
        for (int c = c_lo; c <= c_hi; ++c) {
            const int off = q - c * G * H;
            const int nf = (G < T - c * G) ? G : T - c * G;
            if (off >= 0 && off < (nf - 1) * H + W)
                acc += part[(static_cast<size_t>(g) * nchunks + c) * PL + off];
        }
    return acc / env;
}

// ------------------------------------------------------------------ time-decimated variants (NA = 5)
// The decimated loop carries the waveform only at odd sample indices i = 2v+1 (q = W/2 + i even in hop coordinates),
// stored as xo[v], v in [0, (L-1)/2).  Frame pairs start at even t0, so frame t0 uses the even live samples n' = 2u
// and frame t0+1 the odd ones n' = 2u+1.

// xs[v] = x_padded(q = t0*hop + 2v) for v in [0, W/2 + (hop+1)/2), reflect padding applied on the fly
RF_HD void rf_stage_x_d2(int tid, int nt, float* xs, const float* xo, int L, int t0, int hop) {
    const int nv = RF_PW / 2 + (hop + 1) / 2;
    const int nxo = (L - 1) / 2;
    for (int v = tid; v < nv; v += nt) {
        const int i = rf_reflect_index(t0 * hop + 2 * v - RF_PW / 2, L);   // odd, reflection keeps parity
        const int vo = (i - 1) >> 1;
        xs[v] = (i >= 1 && vo < nxo) ? xo[vo] : 0.f;
    }
}

// decimated overlap-add assembly: waveform sample i = 2v+1 from the half-rate chunk partial sums
// part: [2 groups][nchunks][PLh], chunk c starts at q = c*G*H (even), PLh = ((G-1)*H + W + 1) / 2
RF_HD float rf_ola_sample_d2(int v, const float* part, float env, int G, int PLh, int nchunks, int H, int W) {
    const int q = W / 2 + 2 * v + 1;
    const int cs = G * H;                        // chunk stride in q (even)
    int c_lo = (q - ((G - 1) * H + W) + cs) / cs;  // ceil((q - extent + 1) / cs)
    if (q - ((G - 1) * H + W) + 1 <= 0) c_lo = 0;
    int c_hi = q / cs;
    if (c_hi > nchunks - 1) c_hi = nchunks - 1;
    float acc = 0.f;
    for (int g = 0; g < 2; ++g)
        for (int c = c_lo; c <= c_hi; ++c) {
            const int off = (q - c * cs) >> 1;
            if (off >= 0 && off < PLh) acc += part[(static_cast<size_t>(g) * nchunks + c) * PLh + off];
        }
    return acc / env;
}

// ------------------------------------------------------------------ geometry of the hybrid decimated loop
// Half-rate processing aliases wherever the padded waveform is not band limited: torch.stft's reflect padding puts a
// kink at samples 0 and L-1, measured 3e-3 relative in the first/last five frames and < 1e-7 elsewhere.  The loop
// therefore keeps two full-rate edge strips [0, E) and [L-E, L), E = W + H:
//   * forward STFT: the first 3 frame pairs (frames 0..5) and the pairs from pr_tail = (T-6)/2 on read the strips at
//     full rate, every other pair reads the odd-sample waveform xo;
//   * inverse STFT: the frames that overlap the strips are frames <= 15 (chunk 0) and frames >= T-16 (frame t covers
//     samples [tH - W/2, tH + W/2) and the tail strip starts at (T-1)H - W - H), i.e. chunks >= c_tail = (T-16)/G;
//     those chunks are evaluated a second time on the OTHER sample parity of the half-rate grid (the inverse transform
//     is exact on any sample subset) into `nslots` extra partial-sum slots (slot 0 = chunk 0, slot s = chunk c_tail + s - 1);
//     the two parities interleaved are the full-rate strips.
struct rf_gl_dec_geom {
    int E, pr_tail, c_tail, nslots, n_edge_pairs, nxo;
};
RF_HD rf_gl_dec_geom rf_dec_geom(int T, int G, int H, int W) {
    rf_gl_dec_geom d;
    const int nchunks = (T + G - 1) / G;
    d.E = W + H;
    d.pr_tail = (T - 6) / 2;
    d.c_tail = (T - 16) / G;
    d.nslots = 1 + nchunks - d.c_tail;
    d.n_edge_pairs = 3 + (T + 1) / 2 - d.pr_tail;
    d.nxo = (H * (T - 1) - 1) / 2;
    return d;
}
RF_HD bool rf_dec_ok(int T, int G) { return T >= 4 * G; }

// Edge-strip sample at padded position q = W/2 + i with q ODD (i even) from the other-parity half-rate partial sums of the
// edge chunks (the q-even strip samples are ordinary half-rate samples: rf_ola_sample_d2 with v = (i-1)/2).
// part_o: [2 groups][nslots][PLh], slot 0 = chunk 0, slot s = chunk c_tail + s - 1; position (q - c G H) >> 1 within a chunk.
RF_HD float rf_ola_sample_d2_slots(int q, const float* part_o, float env, int T, int G, int PLh, int c_tail, int nslots,
                                   int H, int W) {
    const int t_hi = (T - 1 < q / H) ? T - 1 : q / H;
    int t_lo = (q - W + H) / H;  // ceil((q-W+1)/H)
    if (q - W + 1 <= 0) t_lo = 0;
    const int c_lo = t_lo / G, c_hi = t_hi / G;
    float acc = 0.f;
    for (int g = 0; g < 2; ++g)
        for (int c = c_lo; c <= c_hi; ++c) {
            if (c != 0 && c < c_tail) continue;      // not an edge chunk: its frames do not reach the strips
            const int slot = c == 0 ? 0 : c - c_tail + 1;
            const int off = (q - c * G * H) >> 1;
            if (slot < nslots && off >= 0 && off < PLh) acc += part_o[(static_cast<size_t>(g) * nslots + slot) * PLh + off];
        }
    return acc / env;
}
