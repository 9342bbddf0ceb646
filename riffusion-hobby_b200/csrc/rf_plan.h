// Host-side plan for path (a): every table the audio kernels read, built in fp64 and
// rounded once to fp32.  Pure C++ (no CUDA) so that tests/hostemu can build it with g++.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "../../include/rf_b200.h"

// Fixed geometry of the prime-factor FFT engine: win = 10*9*49, n_fft = 4*win.
constexpr int RF_W = 4410;
constexpr int RF_N = 4 * RF_W;
constexpr int RF_NA = 10, RF_NB = 9, RF_NC = 49;
constexpr int RF_CHUNK = 16;  // frames per overlap-add chunk in the iSTFT kernel (even)

// Per-bin and per-sample tables in the form the kernels consume them, one set per prime-factor grid (NA = 10: full rate,
// NA = 5: time-decimated loop).  Derived from pp / ph_odd / wt_* below, which stay as the readable (and tested) source.
struct rf_bin_tabs {
    std::vector<uint32_t> bt;      // [n_live] V offset of bin k (s*W + idx) | V offset of its Hermitian partner << 14 | self-paired << 31
    std::vector<float> ab_inv;     // [n_live][4] alpha = conj(ph), beta = i conj(ph) conj(po):  Z[k] = alpha C0 + beta C1
    std::vector<float> ab_fwd;     // [n_live][4] gamma = ph/2, delta = -i ph po/2:  X_t = gamma (Zk + conj Zp), X_t+1 = delta (Zk - conj Zp)
    std::vector<uint32_t> items;   // [49 NA] radix-9 pass: item (a, c) of slot tau as  a*441 + c | n'(a, 0, c) << 12  (rf_pass_b_perm)
    std::vector<float> wg_fwd;     // [9][49 NA][4] per (b, slot): (w0, w1, cos t, -sin t), t = 2 pi n'/N; w0 / w1 = window at the
                                   // sample of frame t0 / t0+1 (NA = 5: the two sample parities, times 2)
    std::vector<float> wg_inv;     // same layout: (w0/N, w1/N, cos t, sin t)
    std::vector<uint16_t> zpos;    // V offsets no live bin or partner of the group writes: [nz[0] entries of group 0 | nz[1] of group 1]
    int nz[2] = {0, 0};
};

struct rf_plan_host {
    rf_plan_desc d{};
    int N = 0, W = 0, H = 0, F = 0, n_mels = 0;
    int n_live = 0, n_even = 0, k_lo = 0, k_hi = 0;

    std::vector<float> window;    // [W] natural order
    std::vector<float> fb;        // [F][n_mels]
    std::vector<int32_t> bins;    // [n_live] private order j -> STFT bin k
    std::vector<int32_t> jofk;    // [F] bin k -> j or -1
    std::vector<uint32_t> pp;     // [n_live] r | idx<<2 | idx2<<15 | (k&7)<<28
    std::vector<float> wt_fwd;    // [4][9][49][10][2]  w[n'] * exp(-2 pi i r n'/N), n' = n_of(a,b,c)
    std::vector<float> wt_inv;    // same layout, w[n']/N * exp(+2 pi i r n'/N)
    // time-decimated Griffin-Lim loop (NA = 5, 2205-point sub-transforms on every second sample); empty if not eligible
    bool decimate = false;
    std::vector<uint32_t> pp2;    // [n_live] like pp with positions on the 5 x 9 x 49 grid and partner 8820 - k
    std::vector<float> wt2_fwd;   // [2 parities][4][9][49][5][2]  2 * w[2u+par] * exp(-2 pi i r u/8820)
    std::vector<float> wt2_inv;   // same layout,                  w[2u+par]/N * exp(+2 pi i r u/8820)
    std::vector<float> ph_odd;    // [n_live][2]  exp(-2 pi i k/N)
    rf_bin_tabs t10, t5;          // kernel-side forms (t5 empty unless `decimate`)
    rf_bin_tabs t5e;              // t5 for the other sample parity (inverse tables ab_inv / wg_inv only differ): the hybrid loop's
                                  // edge chunks run the half-rate inverse transform on both parities instead of a full-rate one
    // mel filterbank in sparse forms over the private bin order
    std::vector<int32_t> melcol_ptr;  // [n_mels+1]  CSR by mel column: entries (j, w)
    std::vector<int32_t> melcol_j;
    std::vector<float> melcol_w;
    std::vector<int32_t> binrow_ptr;  // [n_live+1]  CSR by live bin: entries (m, w)
    std::vector<int32_t> binrow_m;
    std::vector<float> binrow_w;
    // Gram matrix fb^T fb (tridiagonal) and its LU (Thomas) factors, fp64
    std::vector<double> tri;     // [3][n_mels]: sub, diag, super
    std::vector<double> thomas;  // [2][n_mels]: cprime (super/denominator), inv_den
    int fb_nnz = 0;
    // generic engine (any other STFT geometry with n_fft = 2 * (2^a 3^b 5^c 7^d), e.g. 48 kHz: n_fft 19200, 22.05 kHz: 8820):
    // mixed-radix Stockham FFT of n_fft/2 complex points per frame in shared memory; bins in natural order
    bool generic = false;
    bool mixed_radix = false;      // radices / roots2 / rootsN are built: the generic engine and the periodic Griffin-Lim
    std::vector<int> radices;      // product == n_fft / 2
    std::vector<float> roots2;     // [n_fft/2][2]    exp(-2 pi i n / (n_fft/2))
    std::vector<float> rootsN;     // [n_fft/2 + 1][2] exp(-2 pi i k / n_fft)
};

// returns empty string on success, else an error message; `code` gets RF_ERR_*
std::string rf_plan_build_host(const rf_plan_desc& d, const float* window, const float* fb,
                               rf_plan_host& out, int& code);

// PFA index helpers (time side: Ruritanian, spectral side: CRT)
inline int rf_pfa_n_of(int a, int b, int c) { return (441 * a + 490 * b + 90 * c) % RF_W; }
inline int rf_pfa_m_of(int a, int b, int c) { return (441 * a + 3430 * b + 540 * c) % RF_W; }
inline int rf_pfa_pos(int a, int b, int c) { return a * 441 + b * 49 + c; }
// spectral side: the 7-thread radix-49 pass leaves output c of a 49-block at the transposed slot 7 (c % 7) + c / 7
#ifndef RF_GL_PASS7
#define RF_GL_PASS7 1
#endif
inline int rf_pfa_spec_pos(int a, int b, int c) {
    return RF_GL_PASS7 ? a * 441 + b * 49 + 7 * (c % 7) + c / 7 : a * 441 + b * 49 + c;
}
// decimated grid 5 x 9 x 49 (2205 points): time-side index u and the same position formula
inline int rf_pfa2_u_of(int a, int b, int c) { return (441 * a + 245 * b + 45 * c) % 2205; }
