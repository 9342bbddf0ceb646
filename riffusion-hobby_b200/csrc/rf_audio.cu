// Path (a) kernels + C-ABI: STFT / iSTFT / Griffin-Lim / mel / inverse mel / quantisation.
// sm_90a only.  See DESIGN.md §3 for the algorithm and data layout.
#include <cuda_runtime.h>

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

#include "rf_common.h"
#include "rf_generic.cuh"
#include "rf_periodic.cuh"
#include "rf_gl_phases.cuh"
#include "rf_plan.h"
#include "rf_tc.cuh"

// ---------------------------------------------------------------------------------------
// error plumbing
// ---------------------------------------------------------------------------------------
static thread_local std::string g_rf_err;
void rf_set_error(const std::string& msg) { g_rf_err = msg; }
int rf_fail(int code, const std::string& msg) {
    g_rf_err = msg;
    return code;
}
extern "C" const char* rf_last_error(void) { return g_rf_err.c_str(); }
extern "C" const char* rf_version(void) { return "rf_b200 0.1 (sm_90a)"; }

// ---------------------------------------------------------------------------------------
// plan object
// ---------------------------------------------------------------------------------------
struct rf_plan {
    rf_plan_host h;
    std::mutex mu;
    bool uploaded = false;
    int device = -1;
    struct dev_tabs {              // device copies of rf_bin_tabs
        rf_f4* wg_fwd = nullptr;
        rf_f4* wg_inv = nullptr;
        uint32_t* items = nullptr;
        uint32_t* bt = nullptr;
        rf_f4* ab_inv = nullptr;
        rf_f4* ab_fwd = nullptr;
        uint16_t* zpos = nullptr;
    } d10, d5;                     // d5: decimated-loop tables (null when not eligible)
    rf_f4* d5e_wg_inv = nullptr;   // other-parity inverse tables of the decimated grid (rf_plan_host::t5e)
    rf_f4* d5e_ab_inv = nullptr;
    float* d_zero_row = nullptr;   // [n_live] zeros
    int32_t* d_bins = nullptr;
    int32_t* d_jofk = nullptr;
    float* d_win2 = nullptr;
    int32_t* d_melcol_ptr = nullptr;
    int32_t* d_melcol_j = nullptr;
    float* d_melcol_w = nullptr;
    int32_t* d_binrow_ptr = nullptr;
    int32_t* d_binrow_m = nullptr;
    float* d_binrow_w = nullptr;
    double* d_thomas = nullptr;  // [3][n_mels]: sub, cprime, inv_den
    float* d_window = nullptr;    // generic engine
    rf_c32* d_roots2 = nullptr;
    rf_c32* d_rootsN = nullptr;
    bool use_decimation = true;
    std::vector<void*> owned;
};

template <typename T>
static cudaError_t upload(rf_plan* p, T** dst, const void* src, size_t count) {
    cudaError_t e = cudaMalloc(reinterpret_cast<void**>(dst), std::max<size_t>(count, 1) * sizeof(T));
    if (e != cudaSuccess) return e;
    p->owned.push_back(*dst);
    if (count) e = cudaMemcpy(*dst, src, count * sizeof(T), cudaMemcpyHostToDevice);
    return e;
}

static cudaError_t upload_tabs(rf_plan* p, rf_plan::dev_tabs* d, const rf_bin_tabs& t) {
    cudaError_t e = upload(p, &d->wg_fwd, t.wg_fwd.data(), t.wg_fwd.size() / 4);
    if (e == cudaSuccess) e = upload(p, &d->wg_inv, t.wg_inv.data(), t.wg_inv.size() / 4);
    if (e == cudaSuccess) e = upload(p, &d->items, t.items.data(), t.items.size());
    if (e == cudaSuccess) e = upload(p, &d->bt, t.bt.data(), t.bt.size());
    if (e == cudaSuccess) e = upload(p, &d->ab_inv, t.ab_inv.data(), t.ab_inv.size() / 4);
    if (e == cudaSuccess) e = upload(p, &d->ab_fwd, t.ab_fwd.data(), t.ab_fwd.size() / 4);
    if (e == cudaSuccess) e = upload(p, &d->zpos, t.zpos.data(), t.zpos.size());
    return e;
}

static int rf_plan_upload(rf_plan* p) {
    std::lock_guard<std::mutex> lk(p->mu);
    if (p->uploaded) {
        // the tables live on the device that was current at first use: a plan is bound to that device
        int cur = 0;
        RF_CUDA_TRY(cudaGetDevice(&cur));
        if (cur != p->device)
            return rf_fail(RF_ERR_INVALID, "rf_plan: plan tables were uploaded to cuda:" + std::to_string(p->device) +
                                               " but the current device is cuda:" + std::to_string(cur) +
                                               " (create one plan per device)");
        return RF_OK;
    }
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0)
        return rf_fail(RF_ERR_CUDA,
                       "rf_b200: no CUDA device available (this library has no CPU fallback)");
    int dev = 0;
    RF_CUDA_TRY(cudaGetDevice(&dev));
    cudaDeviceProp prop;
    RF_CUDA_TRY(cudaGetDeviceProperties(&prop, dev));
    if (prop.major != 9 || prop.minor != 0)
        return rf_fail(RF_ERR_CUDA, std::string("rf_b200: kernels are built for sm_90a only; device is ") +
                                        prop.name);
    const rf_plan_host& h = p->h;
    RF_CUDA_TRY(upload_tabs(p, &p->d10, h.t10));
    {
        const std::vector<float> zr(h.n_live, 0.f);
        RF_CUDA_TRY(upload(p, &p->d_zero_row, zr.data(), zr.size()));
    }
    RF_CUDA_TRY(upload(p, &p->d_bins, h.bins.data(), h.bins.size()));
    RF_CUDA_TRY(upload(p, &p->d_jofk, h.jofk.data(), h.jofk.size()));
    std::vector<float> w2(h.W);
    for (int i = 0; i < h.W; ++i) w2[i] = h.window[i] * h.window[i];
    RF_CUDA_TRY(upload(p, &p->d_win2, w2.data(), w2.size()));
    RF_CUDA_TRY(upload(p, &p->d_melcol_ptr, h.melcol_ptr.data(), h.melcol_ptr.size()));
    RF_CUDA_TRY(upload(p, &p->d_melcol_j, h.melcol_j.data(), h.melcol_j.size()));
    RF_CUDA_TRY(upload(p, &p->d_melcol_w, h.melcol_w.data(), h.melcol_w.size()));
    RF_CUDA_TRY(upload(p, &p->d_binrow_ptr, h.binrow_ptr.data(), h.binrow_ptr.size()));
    RF_CUDA_TRY(upload(p, &p->d_binrow_m, h.binrow_m.data(), h.binrow_m.size()));
    RF_CUDA_TRY(upload(p, &p->d_binrow_w, h.binrow_w.data(), h.binrow_w.size()));
    std::vector<double> th(3 * static_cast<size_t>(h.n_mels));
    for (int i = 0; i < h.n_mels; ++i) {
        th[i] = h.tri[i];                          // sub
        th[h.n_mels + i] = h.thomas[i];            // cprime
        th[2 * h.n_mels + i] = h.thomas[h.n_mels + i];  // inv_den
    }
    RF_CUDA_TRY(upload(p, &p->d_thomas, th.data(), th.size()));
    if (h.decimate) {
        RF_CUDA_TRY(upload_tabs(p, &p->d5, h.t5));
        RF_CUDA_TRY(upload(p, &p->d5e_wg_inv, h.t5e.wg_inv.data(), h.t5e.wg_inv.size() / 4));
        RF_CUDA_TRY(upload(p, &p->d5e_ab_inv, h.t5e.ab_inv.data(), h.t5e.ab_inv.size() / 4));
    }
    if (h.mixed_radix) {
        RF_CUDA_TRY(upload(p, &p->d_window, h.window.data(), h.window.size()));
        RF_CUDA_TRY(upload(p, &p->d_roots2, h.roots2.data(), h.roots2.size() / 2));
        RF_CUDA_TRY(upload(p, &p->d_rootsN, h.rootsN.data(), h.rootsN.size() / 2));
    }
    p->device = dev;
    p->uploaded = true;
    return RF_OK;
}

extern "C" int rf_plan_create(const rf_plan_desc* desc, const float* window, const float* fb,
                              rf_plan** out) {
    if (!desc || !out) return rf_fail(RF_ERR_INVALID, "rf_plan_create: null argument");
    rf_plan* p = new rf_plan();
    int code = RF_OK;
    std::string err = rf_plan_build_host(*desc, window, fb, p->h, code);
    if (code != RF_OK) {
        delete p;
        return rf_fail(code, err);
    }
    *out = p;
    return RF_OK;
}

extern "C" void rf_plan_destroy(rf_plan* p) {
    if (!p) return;
    for (void* q : p->owned) cudaFree(q);
    delete p;
}

extern "C" int rf_plan_get_info(const rf_plan* p, rf_plan_info* info) {
    if (!p || !info) return rf_fail(RF_ERR_INVALID, "rf_plan_get_info: null argument");
    info->n_freq = p->h.F;
    info->n_live = p->h.n_live;
    info->k_lo = p->h.k_lo;
    info->k_hi = p->h.k_hi;
    info->n_even = p->h.n_even;
    info->fb_nnz = p->h.fb_nnz;
    info->chunk_frames = RF_CHUNK;
    return RF_OK;
}

extern "C" int rf_plan_set_decimation(rf_plan* p, int enable) {
    if (!p) return rf_fail(RF_ERR_INVALID, "rf_plan_set_decimation: null plan");
    p->use_decimation = enable != 0;
    return (p->h.decimate && p->use_decimation) ? 1 : 0;
}

extern "C" int rf_plan_table(const rf_plan* p, const char* name, void* dst, size_t bytes) {
    if (!p || !name || !dst) return rf_fail(RF_ERR_INVALID, "rf_plan_table: null argument");
    const rf_plan_host& h = p->h;
    const void* src = nullptr;
    size_t n = 0;
    std::vector<float> tmp;
    const std::string s(name);
    if (s == "bins") { src = h.bins.data(); n = h.bins.size() * 4; }
    else if (s == "pp") { src = h.pp.data(); n = h.pp.size() * 4; }
    else if (s == "wt_fwd") { src = h.wt_fwd.data(); n = h.wt_fwd.size() * 4; }
    else if (s == "wt_inv") { src = h.wt_inv.data(); n = h.wt_inv.size() * 4; }
    else if (s == "window") { src = h.window.data(); n = h.window.size() * 4; }
    else if (s == "fb") { src = h.fb.data(); n = h.fb.size() * 4; }
    else if (s == "tri") { src = h.tri.data(); n = h.tri.size() * 8; }
    else if (s == "pp2") { src = h.pp2.data(); n = h.pp2.size() * 4; }
    else if (s == "wt2_fwd") { src = h.wt2_fwd.data(); n = h.wt2_fwd.size() * 4; }
    else if (s == "wt2_inv") { src = h.wt2_inv.data(); n = h.wt2_inv.size() * 4; }
    else if (s == "bt") { src = h.t10.bt.data(); n = h.t10.bt.size() * 4; }
    else if (s == "ab_inv") { src = h.t10.ab_inv.data(); n = h.t10.ab_inv.size() * 4; }
    else if (s == "ab_fwd") { src = h.t10.ab_fwd.data(); n = h.t10.ab_fwd.size() * 4; }
    else if (s == "items") { src = h.t10.items.data(); n = h.t10.items.size() * 4; }
    else if (s == "items2") { src = h.t5.items.data(); n = h.t5.items.size() * 4; }
    else if (s == "bt2") { src = h.t5.bt.data(); n = h.t5.bt.size() * 4; }
    else if (s == "ab2_inv") { src = h.t5.ab_inv.data(); n = h.t5.ab_inv.size() * 4; }
    else if (s == "ab2_fwd") { src = h.t5.ab_fwd.data(); n = h.t5.ab_fwd.size() * 4; }
    else if (s == "ph_odd") { src = h.ph_odd.data(); n = h.ph_odd.size() * 4; }
    else if (s == "ab2o_inv") { src = h.t5e.ab_inv.data(); n = h.t5e.ab_inv.size() * 4; }
    else if (s == "wg2_inv") { src = h.t5.wg_inv.data(); n = h.t5.wg_inv.size() * 4; }
    else if (s == "wg2o_inv") { src = h.t5e.wg_inv.data(); n = h.t5e.wg_inv.size() * 4; }
    else if (s == "pinv") {
        // dense min-norm operator P = fb (fb^T fb)^{-1}, built column by column with the
        // same Thomas factors the kernel uses (fp64), for tests
        const int M = h.n_mels;
        std::vector<double> ginv(static_cast<size_t>(M) * M);
        std::vector<double> y(M);
        for (int col = 0; col < M; ++col) {
            for (int i = 0; i < M; ++i) {
                const double rhs = (i == col) ? 1.0 : 0.0;
                y[i] = (rhs - (i ? h.tri[i] * y[i - 1] : 0.0)) * h.thomas[M + i];
            }
            for (int i = M - 2; i >= 0; --i) y[i] -= h.thomas[i] * y[i + 1];
            for (int i = 0; i < M; ++i) ginv[static_cast<size_t>(i) * M + col] = y[i];
        }
        tmp.assign(static_cast<size_t>(h.F) * M, 0.f);
        for (int j = 0; j < h.n_live; ++j) {
            const int k = h.bins[j];
            for (int m = 0; m < M; ++m) {
                double acc = 0;
                for (int e = h.binrow_ptr[j]; e < h.binrow_ptr[j + 1]; ++e)
                    acc += static_cast<double>(h.binrow_w[e]) * ginv[static_cast<size_t>(h.binrow_m[e]) * M + m];
                tmp[static_cast<size_t>(k) * M + m] = static_cast<float>(acc);
            }
        }
        src = tmp.data();
        n = tmp.size() * 4;
    } else
        return rf_fail(RF_ERR_INVALID, "rf_plan_table: unknown table " + s);
    if (n != bytes)
        return rf_fail(RF_ERR_INVALID, "rf_plan_table: size mismatch for " + s + ": have " +
                                           std::to_string(n) + " bytes, caller gave " + std::to_string(bytes));
    std::memcpy(dst, src, n);
    return RF_OK;
}

// ---------------------------------------------------------------------------------------
// kernels
// ---------------------------------------------------------------------------------------

#ifndef RF_GL_PREFETCH
#define RF_GL_PREFETCH 1    // 0: no L2 prefetch of the next pair's rows (A/B builds)
#endif
__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }

// ---- iSTFT of one overlap-add chunk (G frames) of one clip, one r-group ------------------
// Output: dst[PL] partial overlap-add sums of the chunk (NA = 10 full rate, NA = 5 odd samples only).
template <int NA>
__device__ __forceinline__ void istft_chunk_body(unsigned char* smem_raw, const rf_gl_tables& tb,
                                                 const float* __restrict__ S, const rf_c32* __restrict__ cur,
                                                 const rf_c32* __restrict__ prev, int mode, float momentum, int T,
                                                 int G, int PL, int pair_stride, int b, int g, int chunk,
                                                 float* __restrict__ dst) {
    constexpr int W = rf_geom<NA>::W;
    rf_c32* V = reinterpret_cast<rf_c32*>(smem_raw);
    float* ola = reinterpret_cast<float*>(smem_raw + 2 * W * sizeof(rf_c32));
    const int tid = threadIdx.x;
    const int f0 = chunk * G;
    const int nf = min(G, T - f0);
    const int j0 = g ? tb.n_even : 0, j1 = g ? tb.n_live : tb.n_even;
    for (int i = tid; i < PL; i += RF_NT) ola[i] = 0.f;
    const size_t row = static_cast<size_t>(tb.n_live);
    for (int pr = 0; 2 * pr < nf; ++pr) {
        const int t0 = f0 + 2 * pr;
        const bool has1 = (2 * pr + 1) < nf;
        rf_istft_zero<NA>(tid, RF_NT, V, tb, g);
        if (NA == 10) __syncthreads();   // NA = 5 clears only slots the load below does not write
        rf_istft_in in;
        const size_t o0 = (static_cast<size_t>(b) * T + t0) * row;
        in.S0 = S + o0;
        in.cur0 = cur + o0;
        in.prev0 = prev ? prev + o0 : nullptr;
        in.S1 = has1 ? S + o0 + row : tb.zero_row;        // no second frame: zero magnitudes on frame t0's own rows
        in.cur1 = cur + o0 + (has1 ? row : 0);
        in.prev1 = prev ? prev + o0 + (has1 ? row : 0) : nullptr;
        in.mode = mode;
        in.momentum = momentum;
        rf_istft_load<NA>(tid, RF_NT, V, tb, j0, j1, in);
#if RF_GL_PREFETCH
        // the rows of the NEXT pair go to L2 now: its load phase, four FFT passes from here, then waits on L2 instead of HBM
        // (ncu: 37 % of this kernel's samples sat in the load phase, 60 % of them on the long scoreboard)
        if (2 * pr + 2 < nf) {
            const size_t o2 = o0 + 2 * row + j0;
            const int nb4 = (j1 - j0) * 4;   // bytes of a float row segment; the complex rows are twice that
            const int nfr = (2 * pr + 3 < nf) ? 2 : 1;
            for (int f = 0; f < nfr; ++f) {
                const size_t o = o2 + f * row;
                for (int i = tid * 128; i < nb4; i += RF_NT * 128) prefetch_l2(reinterpret_cast<const char*>(S + o) + i);
                for (int i = tid * 128; i < 2 * nb4; i += RF_NT * 128) {
                    prefetch_l2(reinterpret_cast<const char*>(cur + o) + i);
                    if (prev) prefetch_l2(reinterpret_cast<const char*>(prev + o) + i);
                }
            }
        }
#endif
        __syncthreads();
        rf_pass_c7<true, NA, 0>(tid, RF_NT, V);
        __syncthreads();
        rf_pass_c7<true, NA, 1>(tid, RF_NT, V);
        __syncthreads();
        rf_pass_a<true, NA>(tid, RF_NT, V);
        __syncthreads();
        rf_istft_pass_b<NA>(tid, RF_NT, V, ola + pr * pair_stride, tb, g, has1, 2);
        __syncthreads();
    }
    for (int i = tid; i < PL; i += RF_NT) dst[i] = ola[i];
}

// full rate: grid (nchunks*2, B), part[b][g][chunk][PL]
__global__ void __launch_bounds__(RF_NT, 2)
k_istft_chunk(rf_gl_tables tb, const float* __restrict__ S, const rf_c32* __restrict__ cur,
              const rf_c32* __restrict__ prev, int mode, float momentum, int T, int G, int PL, int nchunks,
              float* __restrict__ part) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int g = blockIdx.x & 1, chunk = blockIdx.x >> 1, b = blockIdx.y;
    istft_chunk_body<10>(smem_raw, tb, S, cur, prev, mode, momentum, T, G, PL, 2 * tb.off1, b, g, chunk,
                         part + ((static_cast<size_t>(b) * 2 + g) * nchunks + chunk) * PL);
}

// hybrid decimated loop (rf_gl_dec_geom): grid ((nchunks + nslots) * 2, B)
//   blocks [0, nchunks*2): half-rate partial sums of every chunk (part_h[b][g][chunk][PLh]): the waveform samples at even
//                 padded positions q (odd sample index i).  2205-point sub-transforms: 57 KB of shared memory and <= 85
//                 registers with the 7-thread radix-49 pass -> 3 CTAs/SM
//   blocks behind: the edge chunks (slot 0 = chunk 0, slot s = chunk c_tail + s - 1) once more on the OTHER sample parity
//                 (tables tbo: frame t0 takes the odd live samples, frame t0+1 the even ones) -> part_o[b][g][slot][PLh],
//                 the samples at odd q.  Together the two parities are the full-rate edge strips: the inverse transform of a
//                 band-limited spectrum is exact on any sample subset, so nothing aliases here (the forward side is where
//                 the strips are needed).  Round 2's separate full-rate launch for these chunks (112 KB, 2 CTAs/SM, one
//                 under-filled wave of long CTAs: 0.2 ms of every iteration) is gone.
#ifndef RF_GL_HALF_MINB
#define RF_GL_HALF_MINB 3   // CTAs per SM the half-rate kernels are compiled for (A/B builds: 2)
#endif
__global__ void __launch_bounds__(RF_NT, RF_GL_HALF_MINB)
k_istft_half(rf_gl_tables tb2, rf_gl_tables tbo, const float* __restrict__ S, const rf_c32* __restrict__ cur,
             const rf_c32* __restrict__ prev, int mode, float momentum, int T, int G, int PLh, int nchunks, int c_tail,
             int nslots, float* __restrict__ part_h, float* __restrict__ part_o) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int g = blockIdx.x & 1, b = blockIdx.y, idx = blockIdx.x >> 1;
    const bool other = idx >= nchunks;                       // an edge chunk on the other sample parity
    const int slot = idx - nchunks;
    const int chunk = !other ? idx : (slot == 0 ? 0 : c_tail + slot - 1);
    float* dst = !other ? part_h + ((static_cast<size_t>(b) * 2 + g) * nchunks + idx) * PLh
                        : part_o + ((static_cast<size_t>(b) * 2 + g) * nslots + slot) * PLh;
    rf_gl_tables tb = tb2;                                   // the two table sets differ in three fields
    if (other) {
        tb.wg_inv = tbo.wg_inv;
        tb.ab_inv = tbo.ab_inv;
        tb.off1 = tbo.off1;
    }
    istft_chunk_body<5>(smem_raw, tb, S, cur, prev, mode, momentum, T, G, PLh, 441, b, g, chunk, dst);
}

// ---- overlap-add assembly: x[b][i] = sum(parts) / envelope, kept region only --------------
// (torch.istft: y / window_envelope, trimmed by n_fft/2 each side)
__global__ void k_envelope(const float* __restrict__ win2, int T, int H, int W, int L, float* __restrict__ env) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < L) env[i] = rf_envelope(i, win2, T, H, W);
}

__global__ void k_ola_assemble(const float* __restrict__ part, const float* __restrict__ env,
                               int T, int G, int PL, int nchunks, int H, int W, int L,
                               float* __restrict__ x) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.y;
    if (i >= L) return;
    x[static_cast<size_t>(b) * L + i] =
        rf_ola_sample(i, part + static_cast<size_t>(b) * 2 * nchunks * PL, env[i], T, G, PL, nchunks, H, W);
}

// decimated assembly: xd[b] = [ xo (nxo odd samples 2v+1) | head strip x[0..E) | tail strip x[L-E..L) ]
// strip sample i sits at padded position q = W/2 + i: even q = an ordinary half-rate sample, odd q from the other-parity
// partial sums of the edge chunks.  The decimated loop only exists for hop 441 / win 4410 / 16-frame chunks
// (rf_plan_build_host): compile-time constants turn the index divisions into multiplies.
// (two kernels: the strip samples need frame-accurate chunk bounds and twice the registers; kept out of the streaming one)
__global__ void k_ola_assemble_dec(const float* __restrict__ part_h, const float* __restrict__ env, int PLh, int nchunks,
                                   int nxo, int E, float* __restrict__ xd) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.y;
    if (v >= nxo) return;
    xd[static_cast<size_t>(b) * (nxo + 2 * E) + v] =
        rf_ola_sample_d2(v, part_h + static_cast<size_t>(b) * 2 * nchunks * PLh, env[2 * v + 1], RF_CHUNK, PLh, nchunks, 441,
                         RF_PW);
}
__global__ void k_ola_assemble_strips(const float* __restrict__ part_h, const float* __restrict__ part_o,
                                      const float* __restrict__ env, int T, int PLh, int nchunks, int c_tail, int nslots,
                                      int L, int nxo, int E, float* __restrict__ xd) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.y;
    if (e >= 2 * E) return;
    const int i = e < E ? e : L - 2 * E + e;
    float r;
    if (i & 1)
        r = rf_ola_sample_d2((i - 1) >> 1, part_h + static_cast<size_t>(b) * 2 * nchunks * PLh, env[i], RF_CHUNK, PLh, nchunks,
                             441, RF_PW);
    else
        r = rf_ola_sample_d2_slots(RF_PW / 2 + i, part_o + static_cast<size_t>(b) * 2 * nslots * PLh, env[i], T, RF_CHUNK, PLh,
                                   c_tail, nslots, 441, RF_PW);
    xd[static_cast<size_t>(b) * (nxo + 2 * E) + nxo + e] = r;
}

// 1-D TMA bulk copy of n floats starting at src (any 4-byte alignment) into shared memory: the copy starts at the enclosing
// 16-byte boundary and is rounded up to 16 bytes — the caller guarantees those few extra bytes are readable — and lands at
// xs_al (16-byte aligned); src[0] ends up bulk_shift(src) bytes behind xs_al.  One thread issues; completion on `bar`.
__device__ __forceinline__ uint32_t bulk_shift(const float* src) {
    return static_cast<uint32_t>(reinterpret_cast<uint64_t>(src) & 15u);
}
__device__ __forceinline__ void bulk_issue(float* xs_al, uint64_t* bar, const float* src, int n) {
    const uint64_t a = reinterpret_cast<uint64_t>(src);
    const uint32_t shift = static_cast<uint32_t>(a & 15u);
    const uint32_t nbytes = (shift + static_cast<uint32_t>(n) * 4u + 15u) & ~15u;
    tc::mbar_expect_tx(bar, nbytes);
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     tc::smem_u32(xs_al)),
                 "l"(a - shift), "r"(nbytes), "r"(tc::smem_u32(bar))
                 : "memory");
}
// staging buffer of the half-rate STFT CTAs: W/2 + (hop+1)/2 samples + up to 3 floats of alignment slack, rounded to 16
// bytes.  Two of them (double buffering over the CTA's pairs), then the two mbarriers.
constexpr int RF_XS_HALF_N = RF_PW / 2 + (441 + 1) / 2;
constexpr int RF_XS_HALF_BYTES = ((RF_XS_HALF_N + 3) * 4 + 15) / 16 * 16;
constexpr int RF_STFT_HALF_PAIRS = 4;    // consecutive frame pairs per half-rate STFT CTA

// ---- STFT of one frame pair, one r-group ------------------------------------------------
// x_full: waveform holding samples [base, ...) (reflect padding applied on the fly); NA = 5: xo odd samples
template <int NA>
__device__ __forceinline__ void stft_pair_body(unsigned char* smem_raw, const rf_gl_tables& tb,
                                               const float* __restrict__ x, int base, int L, int T, int hop, int b,
                                               int g, int pr, rf_c32* __restrict__ R) {
    constexpr int W = rf_geom<NA>::W;
    rf_c32* V = reinterpret_cast<rf_c32*>(smem_raw);
    float* xs = reinterpret_cast<float*>(smem_raw + 2 * W * sizeof(rf_c32));
    const int tid = threadIdx.x;
    const int t0 = 2 * pr;
    const bool has1 = t0 + 1 < T;
    if (NA == 10) rf_stage_x(tid, RF_NT, xs, x, L, t0, hop, base);
    else rf_stage_x_d2(tid, RF_NT, xs, x, L, t0, hop);
    __syncthreads();
    rf_stft_pass_b<NA>(tid, RF_NT, V, xs, tb, g, has1);
    __syncthreads();
    rf_pass_a<false, NA>(tid, RF_NT, V);
    __syncthreads();
    rf_pass_c7<false, NA, 0>(tid, RF_NT, V);
    __syncthreads();
    rf_pass_c7<false, NA, 1>(tid, RF_NT, V);
    __syncthreads();
    const int j0 = g ? tb.n_even : 0, j1 = g ? tb.n_live : tb.n_even;
    rf_c32* out0 = R + (static_cast<size_t>(b) * T + t0) * tb.n_live;
    rf_stft_post<NA>(tid, RF_NT, V, tb, j0, j1, out0, has1 ? out0 + tb.n_live : nullptr);
}

// full rate: grid (npairs*2, B). x: [B][L] un-padded signal
__global__ void __launch_bounds__(RF_NT, 2)
k_stft_pair(rf_gl_tables tb, const float* __restrict__ x, int L, int T, int hop, rf_c32* __restrict__ R) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int g = blockIdx.x & 1, pr = blockIdx.x >> 1, b = blockIdx.y;
    stft_pair_body<10>(smem_raw, tb, x + static_cast<size_t>(b) * L, 0, L, T, hop, b, g, pr, R);
}

// hybrid decimated loop, two launches: k_stft_edge, grid (n_edge_pairs*2, B): the edge pairs (3 head pairs, then the
// pairs from pr_tail on) at full rate from the strips of xd; k_stft_half, grid ((npairs - n_edge_pairs)*2, B): the rest
// from the odd samples xo at half rate (55 KB of shared memory with the two TMA staging buffers, <= 85 registers: 3 CTAs/SM)
__global__ void __launch_bounds__(RF_NT, 2)
k_stft_edge(rf_gl_tables tb, const float* __restrict__ xd, int L, int T, int hop, int nxo, int E, int pr_tail,
            rf_c32* __restrict__ R) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int g = blockIdx.x & 1, b = blockIdx.y;
    const int idx = blockIdx.x >> 1;
    const float* xb = xd + static_cast<size_t>(b) * (nxo + 2 * E);
    if (idx < 3) stft_pair_body<10>(smem_raw, tb, xb + nxo, 0, L, T, hop, b, g, idx, R);
    else stft_pair_body<10>(smem_raw, tb, xb + nxo + E, L - E, L, T, hop, b, g, pr_tail + idx - 3, R);
}

// Half-rate pairs never touch the reflect padding (the hybrid loop gives those to k_stft_edge), so the samples of a pair
// are RF_XS_HALF_N consecutive odd samples xo[vo0 ..): ONE 1-D TMA bulk copy per pair instead of a load loop, and a CTA takes
// RF_STFT_HALF_PAIRS consecutive pairs [pr_lo + P i, ..) < pr_hi so that the copy of the next pair flies during the four
// passes of the current one (two staging buffers, one mbarrier each).
#ifndef RF_STFT_HALF_MINB
#define RF_STFT_HALF_MINB RF_GL_HALF_MINB   // 4 fits the shared memory (4 x 54.7 KB) but needs <= 64 registers (A/B builds)
#endif
__global__ void __launch_bounds__(RF_NT, RF_STFT_HALF_MINB)
k_stft_half(rf_gl_tables tb2, const float* __restrict__ xd, int L, int T, int hop, int nxo, int E, int pr_lo, int pr_hi,
            rf_c32* __restrict__ R) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    constexpr int W = rf_geom<5>::W;
    const int g = blockIdx.x & 1, b = blockIdx.y, tid = threadIdx.x;
    const float* xo = xd + static_cast<size_t>(b) * (nxo + 2 * E);
    rf_c32* V = reinterpret_cast<rf_c32*>(smem_raw);
    unsigned char* xbuf = smem_raw + 2 * W * sizeof(rf_c32);
    uint64_t* bars = reinterpret_cast<uint64_t*>(xbuf + 2 * RF_XS_HALF_BYTES);
    const int first = pr_lo + (blockIdx.x >> 1) * RF_STFT_HALF_PAIRS;
    const int npr = min(RF_STFT_HALF_PAIRS, pr_hi - first);
    auto src_of = [&](int pr) { return xo + ((2 * pr * hop - RF_PW / 2 - 1) >> 1); };
    if (tid == 0) {
        tc::mbar_init(&bars[0], 1);
        tc::mbar_init(&bars[1], 1);
        tc::fence_barrier_init();
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        bulk_issue(reinterpret_cast<float*>(xbuf), &bars[0], src_of(first), RF_XS_HALF_N);
    }
    __syncthreads();   // the initialised barriers are visible to every thread before it waits
    const int j0 = g ? tb2.n_even : 0, j1 = g ? tb2.n_live : tb2.n_even;
    for (int i = 0; i < npr; ++i) {
        const int pr = first + i, t0 = 2 * pr;
        const bool has1 = t0 + 1 < T;
        // buffer (i+1)&1 was last read by the radix-9 pass of pair i-1, which every thread left at least one barrier ago
        if (tid == 0 && i + 1 < npr)
            bulk_issue(reinterpret_cast<float*>(xbuf + ((i + 1) & 1) * RF_XS_HALF_BYTES), &bars[(i + 1) & 1], src_of(pr + 1),
                       RF_XS_HALF_N);
        tc::mbar_wait(&bars[i & 1], (i >> 1) & 1);
        const float* xs = reinterpret_cast<const float*>(xbuf + (i & 1) * RF_XS_HALF_BYTES + bulk_shift(src_of(pr)));
        rf_stft_pass_b<5>(tid, RF_NT, V, xs, tb2, g, has1);
        __syncthreads();
        rf_pass_a<false, 5>(tid, RF_NT, V);
        __syncthreads();
        rf_pass_c7<false, 5, 0>(tid, RF_NT, V);
        __syncthreads();
        rf_pass_c7<false, 5, 1>(tid, RF_NT, V);
        __syncthreads();
        rf_c32* out0 = R + (static_cast<size_t>(b) * T + t0) * tb2.n_live;
        rf_stft_post<5>(tid, RF_NT, V, tb2, j0, j1, out0, has1 ? out0 + tb2.n_live : nullptr);
        __syncthreads();   // V is rewritten by the next pair
    }
}

// ---- STFT + |.| + mel of one frame pair (both groups in one CTA) -------------------------
__global__ void __launch_bounds__(RF_NT, 1)
k_stft_mel_pair(rf_gl_tables tb, const float* __restrict__ x, int L, int T, int n_mels,
                const int32_t* __restrict__ melcol_ptr, const int32_t* __restrict__ melcol_j,
                const float* __restrict__ melcol_w, float* __restrict__ mel) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    rf_c32* V = reinterpret_cast<rf_c32*>(smem_raw);
    float* xs = reinterpret_cast<float*>(smem_raw + 2 * RF_PW * sizeof(rf_c32));
    rf_c32* spec0 = reinterpret_cast<rf_c32*>(xs + RF_PW + tb.off1 + ((RF_PW + tb.off1) & 1));
    rf_c32* spec1 = spec0 + tb.n_live;
    const int tid = threadIdx.x;
    const int pr = blockIdx.x, b = blockIdx.y;
    const int t0 = 2 * pr;
    const bool has1 = t0 + 1 < T;
    rf_stage_x(tid, RF_NT, xs, x + static_cast<size_t>(b) * L, L, t0, tb.off1);
    __syncthreads();
    for (int g = 0; g < 2; ++g) {
        rf_stft_pass_b<10>(tid, RF_NT, V, xs, tb, g, has1);
        __syncthreads();
        rf_pass_a<false, 10>(tid, RF_NT, V);
        __syncthreads();
        rf_pass_c7<false, 10, 0>(tid, RF_NT, V);
        __syncthreads();
        rf_pass_c7<false, 10, 1>(tid, RF_NT, V);
        __syncthreads();
        const int j0 = g ? tb.n_even : 0, j1 = g ? tb.n_live : tb.n_even;
        rf_stft_post<10>(tid, RF_NT, V, tb, j0, j1, spec0, spec1);
        __syncthreads();
    }
    // magnitude in place (spec.x = |X|), torch.abs on complex64
    for (int j = tid; j < tb.n_live; j += RF_NT) {
        spec0[j].x = hypotf(spec0[j].x, spec0[j].y);
        spec1[j].x = hypotf(spec1[j].x, spec1[j].y);
    }
    __syncthreads();
    // mel[m] = sum_k fb[k][m] |X[k]|   (MelScale.forward, TA/transforms/_transforms.py:417)
    for (int it = tid; it < 2 * n_mels; it += RF_NT) {
        const int f = it / n_mels, m = it - f * n_mels;
        if (f == 1 && !has1) continue;
        const rf_c32* sp = f ? spec1 : spec0;
        float acc = 0.f;
        for (int e = melcol_ptr[m]; e < melcol_ptr[m + 1]; ++e) acc += melcol_w[e] * sp[melcol_j[e]].x;
        mel[(static_cast<size_t>(b) * n_mels + m) * T + t0 + f] = acc;
    }
}

// ---- layout permutations between torchaudio's [B][F][T] and the private [B][T][n_live] ----
template <typename TT>
__global__ void k_gather_FT_to_TJ(const TT* __restrict__ src, const int32_t* __restrict__ bins,
                                  int F, int T, int n_live, TT* __restrict__ dst) {
    __shared__ TT tile[32][33];
    const int b = blockIdx.z;
    const int j0 = blockIdx.x * 32, t0 = blockIdx.y * 32;
    {
        const int j = j0 + threadIdx.y, t = t0 + threadIdx.x;
        if (j < n_live && t < T)
            tile[threadIdx.y][threadIdx.x] = src[(static_cast<size_t>(b) * F + bins[j]) * T + t];
    }
    __syncthreads();
    {
        const int t = t0 + threadIdx.y, j = j0 + threadIdx.x;
        if (j < n_live && t < T)
            dst[(static_cast<size_t>(b) * T + t) * n_live + j] = tile[threadIdx.x][threadIdx.y];
    }
}

template <typename TT>
__global__ void k_scatter_TJ_to_FT(const TT* __restrict__ src, const int32_t* __restrict__ bins,
                                   int F, int T, int n_live, TT* __restrict__ dst) {
    __shared__ TT tile[32][33];
    const int b = blockIdx.z;
    const int j0 = blockIdx.x * 32, t0 = blockIdx.y * 32;
    {
        const int t = t0 + threadIdx.y, j = j0 + threadIdx.x;
        if (j < n_live && t < T)
            tile[threadIdx.y][threadIdx.x] = src[(static_cast<size_t>(b) * T + t) * n_live + j];
    }
    __syncthreads();
    {
        const int j = j0 + threadIdx.y, t = t0 + threadIdx.x;
        if (j < n_live && t < T)
            dst[(static_cast<size_t>(b) * F + bins[j]) * T + t] = tile[threadIdx.x][threadIdx.y];
    }
}

__global__ void k_fill_c32(rf_c32* p, size_t n, float re, float im) {
    const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i < n) p[i] = c_make(re, im);
}

// ---- inverse mel: relu(fb (fb^T fb)^-1 mel) per time column -------------------------------
// CTA = 32 time columns of one clip.  Phase 1: stage mel[:, t0:t0+32] in smem.  Phase 2: warp 0
// solves the tridiagonal system per column in fp64 (Thomas).  Phase 3: sparse fb apply + relu.
// out_mode 0: S[b][t][j] (private), 1: lin[b][k][t] (torchaudio layout; dead rows pre-zeroed)
__global__ void __launch_bounds__(256)
k_inverse_mel(const float* __restrict__ mel, int T, int n_mels, int n_live, int F,
              const double* __restrict__ thomas, const int32_t* __restrict__ binrow_ptr,
              const int32_t* __restrict__ binrow_m, const float* __restrict__ binrow_w,
              const int32_t* __restrict__ bins, int out_mode, float* __restrict__ out) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float* ys = reinterpret_cast<float*>(smem_raw);  // [n_mels][33]
    const int b = blockIdx.y, t0 = blockIdx.x * 32;
    const int tid = threadIdx.x;
    for (int i = tid; i < n_mels * 32; i += blockDim.x) {
        const int m = i >> 5, tl = i & 31;
        ys[m * 33 + tl] = (t0 + tl < T) ? mel[(static_cast<size_t>(b) * n_mels + m) * T + t0 + tl] : 0.f;
    }
    __syncthreads();
    if (tid < 32) {
        const double* sub = thomas;
        const double* cp = thomas + n_mels;
        const double* idn = thomas + 2 * n_mels;
        double prevv = 0.0;
        for (int m = 0; m < n_mels; ++m) {
            const double v = (static_cast<double>(ys[m * 33 + tid]) - sub[m] * prevv) * idn[m];
            ys[m * 33 + tid] = static_cast<float>(v);  // forward sweep kept in fp32 storage
            prevv = v;
        }
        // back substitution: re-run in fp64 from the stored forward values
        double nxt = static_cast<double>(ys[(n_mels - 1) * 33 + tid]);
        for (int m = n_mels - 2; m >= 0; --m) {
            const double v = static_cast<double>(ys[m * 33 + tid]) - cp[m] * nxt;
            ys[m * 33 + tid] = static_cast<float>(v);
            nxt = v;
        }
    }
    __syncthreads();
    if (out_mode == 0) {
        // bin outer, time inner: a live bin touches at most two filters (tridiagonal Gram), so its (filter, weight) pairs
        // are fetched once and reused for the 32 time columns; for each column consecutive threads write consecutive bins
        const int nt = min(32, T - t0);
        float* base = out + (static_cast<size_t>(b) * T + t0) * n_live;
        for (int j = tid; j < n_live; j += blockDim.x) {
            const int e0 = binrow_ptr[j], e1 = binrow_ptr[j + 1];
            if (e1 - e0 <= 2) {
                const float w0 = e1 > e0 ? binrow_w[e0] : 0.f, w1 = e1 > e0 + 1 ? binrow_w[e0 + 1] : 0.f;
                const float* y0 = ys + (e1 > e0 ? binrow_m[e0] : 0) * 33;
                const float* y1 = ys + (e1 > e0 + 1 ? binrow_m[e0 + 1] : 0) * 33;
                for (int tl = 0; tl < nt; ++tl)
                    base[static_cast<size_t>(tl) * n_live + j] = fmaxf(fmaf(w1, y1[tl], w0 * y0[tl]), 0.f);
            } else {
                for (int tl = 0; tl < nt; ++tl) {
                    float acc = 0.f;
                    for (int e = e0; e < e1; ++e) acc += binrow_w[e] * ys[binrow_m[e] * 33 + tl];
                    base[static_cast<size_t>(tl) * n_live + j] = fmaxf(acc, 0.f);
                }
            }
        }
    } else {
        const int tl = tid & 31;
        for (int j = tid >> 5; j < n_live; j += blockDim.x >> 5) {
            float acc = 0.f;
            for (int e = binrow_ptr[j]; e < binrow_ptr[j + 1]; ++e)
                acc += binrow_w[e] * ys[binrow_m[e] * 33 + tl];
            if (t0 + tl < T) out[(static_cast<size_t>(b) * F + bins[j]) * T + t0 + tl] = fmaxf(acc, 0.f);
        }
    }
}

// ---- MelScale on its own: mel[b][m][t] = sum_k fb[k][m] spec[b][k][t] ---------------------
__global__ void k_mel_scale(const float* __restrict__ spec, int F, int T, int n_mels,
                            const int32_t* __restrict__ melcol_ptr, const int32_t* __restrict__ melcol_j,
                            const float* __restrict__ melcol_w, const int32_t* __restrict__ bins,
                            float* __restrict__ mel) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    const int m = blockIdx.y, b = blockIdx.z;
    if (t >= T) return;
    float acc = 0.f;
    for (int e = melcol_ptr[m]; e < melcol_ptr[m + 1]; ++e)
        acc += melcol_w[e] * spec[(static_cast<size_t>(b) * F + bins[melcol_j[e]]) * T + t];
    mel[(static_cast<size_t>(b) * n_mels + m) * T + t] = acc;
}

// ---- image <-> mel quantisation, int16 -------------------------------------------------------
__global__ void k_image_to_mel(const uint8_t* __restrict__ img, int Hh, int Ww, int stereo, float inv_power,
                               float max_value, float* __restrict__ mel) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y;  // output row (mel bin, 0 = lowest) = image row Hh-1-y
    const int c = blockIdx.z;
    if (x >= Ww) return;
    const int plane = stereo ? (1 + c) : 0;
    const uint8_t u = img[(static_cast<size_t>(Hh - 1 - y) * Ww + x) * 3 + plane];
    float d = 255.0f - static_cast<float>(u);
    d = d / 255.0f;
    d = powf(d, inv_power);
    mel[(static_cast<size_t>(c) * Hh + y) * Ww + x] = d * max_value;
}

__global__ void k_absmax(const float* __restrict__ v, size_t n, int use_abs, float* __restrict__ out) {
    float m = 0.f;
    for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
         i += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const float a = use_abs ? fabsf(v[i]) : v[i];
        m = fmaxf(m, a);
    }
    for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    // values are >= 0 so the int ordering of the bit patterns equals the float ordering
    if ((threadIdx.x & 31) == 0) atomicMax(reinterpret_cast<int*>(out), __float_as_int(m));
}

__global__ void k_mel_to_image(const float* __restrict__ mel, int C, int Hh, int Ww, float power,
                               const float* __restrict__ maxv, uint8_t* __restrict__ img) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y;  // image row
    if (x >= Ww) return;
    const float mx = *maxv;
    uint8_t px[3];
    for (int c = 0; c < C; ++c) {
        float d = mel[(static_cast<size_t>(c) * Hh + (Hh - 1 - y)) * Ww + x] / mx;
        d = powf(d, power);
        d = d * 255.0f;
        d = 255.0f - d;
        px[c] = static_cast<uint8_t>(d);  // truncation (numpy astype(uint8) on [0,255])
    }
    uint8_t* o = img + (static_cast<size_t>(y) * Ww + x) * 3;
    if (C == 1) {
        o[0] = o[1] = o[2] = px[0];
    } else {
        o[0] = 0;
        o[1] = px[0];
        o[2] = px[1];
    }
}

__global__ void k_wave_to_int16(const float* __restrict__ w, int C, int L, const float* __restrict__ maxv,
                                int normalize, int16_t* __restrict__ pcm) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= L) return;
    // samples *= iinfo(int16).max / max|samples|  (audio_util.py:24): the scale is computed in
    // fp32 (numpy float32 scalar arithmetic), then multiplied.
    const float scale = normalize ? (32767.0f / *maxv) : 1.0f;
    for (int c = 0; c < C; ++c) {
        const float v = w[static_cast<size_t>(c) * L + i] * scale;
        pcm[static_cast<size_t>(i) * C + c] = static_cast<int16_t>(v);  // truncation toward zero
    }
}

// ---------------------------------------------------------------------------------------
// host drivers
// ---------------------------------------------------------------------------------------
static rf_gl_tables make_tables(const rf_plan* p, int NA = 10) {
    rf_gl_tables tb;
    const rf_plan::dev_tabs& d = NA == 10 ? p->d10 : p->d5;
    const rf_bin_tabs& t = NA == 10 ? p->h.t10 : p->h.t5;
    tb.wg_fwd = d.wg_fwd;
    tb.wg_inv = d.wg_inv;
    tb.items = d.items;
    tb.bt = d.bt;
    tb.ab_inv = d.ab_inv;
    tb.ab_fwd = d.ab_fwd;
    tb.zpos = d.zpos;
    tb.nz0 = t.nz[0];
    tb.nz1 = t.nz[1];
    tb.zero_row = p->d_zero_row;
    tb.off1 = NA == 10 ? p->h.H : (p->h.H + 1) / 2;
    tb.n_live = p->h.n_live;
    tb.n_even = p->h.n_even;
    return tb;
}

static rf_gen_tab make_gen_tab(const rf_plan* p) {
    rf_gen_tab g{};
    g.roots2 = p->d_roots2;
    g.rootsN = p->d_rootsN;
    g.window = p->d_window;
    g.bins = p->d_bins;
    g.N = p->h.N;
    g.N2 = p->h.N / 2;
    g.W = p->h.W;
    g.H = p->h.H;
    g.lo = (p->h.N - p->h.W) / 2;
    g.J = p->h.n_live;
    g.nrad = static_cast<int>(p->h.radices.size());
    for (int i = 0; i < g.nrad; ++i) g.rad[i] = p->h.radices[i];
    return g;
}
static size_t gen_smem(const rf_plan* p) { return (2 * static_cast<size_t>(p->h.N / 2) + 2) * sizeof(rf_c32); }
static int gen_smem_attrs(const rf_plan* p) {
    static rf_dev_once once[2];
    const int bytes = static_cast<int>(gen_smem(p));
    if (bytes > 227 * 1024) return rf_fail(RF_ERR_UNSUPPORTED, "generic FFT engine: n_fft too large for shared memory");
    cudaError_t err = rf_set_smem_once(once[0], k_gen_stft, 227 * 1024);
    if (err == cudaSuccess) err = rf_set_smem_once(once[1], k_gen_istft, 227 * 1024);
    if (err != cudaSuccess) return rf_fail(RF_ERR_CUDA, std::string("cudaFuncSetAttribute: ") + cudaGetErrorString(err));
    return RF_OK;
}

static size_t align256(size_t v) { return (v + 255) & ~static_cast<size_t>(255); }

struct gl_ws {
    float* S;
    rf_c32* R[2];
    float* part;
    float* env;
    float* part_e;  // decimated loop: other-parity half-rate partial sums of the edge chunks [B][2][nslots][PLh]
    float* xd;      // decimated loop: [B][nxo + 2E] odd samples + the two full-rate edge strips
    size_t total;
    int nchunks, PL;
};

static gl_ws gl_layout(const rf_plan* p, int B, int T, void* base) {
    gl_ws w;
    const size_t bt = static_cast<size_t>(B) * T * p->h.n_live;
    w.nchunks = (T + RF_CHUNK - 1) / RF_CHUNK;
    w.PL = (RF_CHUNK - 1) * p->h.H + p->h.W;
    size_t off = 0;
    unsigned char* b = static_cast<unsigned char*>(base);
    w.S = reinterpret_cast<float*>(b + off);
    off += align256(bt * 4);
    w.R[0] = reinterpret_cast<rf_c32*>(b + off);
    off += align256(bt * 8);
    w.R[1] = reinterpret_cast<rf_c32*>(b + off);
    off += align256(bt * 8);
    w.part = reinterpret_cast<float*>(b + off);
    if (p->h.generic) off += align256(static_cast<size_t>(B) * T * p->h.W * 4);      // windowed frames [B][T][W]
    else off += align256(static_cast<size_t>(B) * 2 * w.nchunks * w.PL * 4);
    w.env = reinterpret_cast<float*>(b + off);
    off += align256(static_cast<size_t>(p->h.H) * (T > 0 ? T - 1 : 0) * 4);
    w.part_e = w.xd = nullptr;
    if (p->h.decimate && rf_dec_ok(T, RF_CHUNK)) {
        const rf_gl_dec_geom d = rf_dec_geom(T, RF_CHUNK, p->h.H, p->h.W);
        w.part_e = reinterpret_cast<float*>(b + off);
        off += align256(static_cast<size_t>(B) * 2 * d.nslots * ((w.PL + 1) / 2) * 4);
        w.xd = reinterpret_cast<float*>(b + off);
        off += align256(static_cast<size_t>(B) * (d.nxo + 2 * d.E) * 4);
    }
    w.total = off;
    return w;
}

extern "C" size_t rf_griffinlim_workspace_bytes(const rf_plan* p, int B, int T) {
    if (!p || B <= 0 || T <= 0) return 0;
    return gl_layout(p, B, T, nullptr).total;
}

static int check_T(const rf_plan* p, int T, const char* who) {
    const int L = p->h.H * (T - 1);
    if (T < 1 || L <= p->h.N / 2)
        return rf_fail(RF_ERR_INVALID,
                       std::string(who) + ": Padding size should be less than the corresponding input "
                       "dimension (hop*(T-1) = " + std::to_string(L) + " must exceed n_fft/2 = " +
                           std::to_string(p->h.N / 2) + ")");
    return RF_OK;
}

static int set_smem_attrs() {
    static rf_dev_once once[8];
    cudaError_t err = rf_set_smem_once(once[0], k_istft_chunk, 200 * 1024);
    if (err == cudaSuccess) err = rf_set_smem_once(once[6], k_istft_half, 200 * 1024);
    if (err == cudaSuccess) err = rf_set_smem_once(once[7], k_stft_half, 200 * 1024);
    if (err == cudaSuccess) err = rf_set_smem_once(once[2], k_stft_pair, 200 * 1024);
    if (err == cudaSuccess) err = rf_set_smem_once(once[3], k_stft_edge, 200 * 1024);
    if (err == cudaSuccess) err = rf_set_smem_once(once[4], k_stft_mel_pair, 227 * 1024);
    if (err == cudaSuccess) err = rf_set_smem_once(once[5], k_inverse_mel, 200 * 1024);
    if (err != cudaSuccess) return rf_fail(RF_ERR_CUDA, std::string("cudaFuncSetAttribute: ") + cudaGetErrorString(err));
    return RF_OK;
}

static int launch_inverse_mel(rf_plan* p, const float* d_mel, int B, int T, int out_mode, float* out,
                              cudaStream_t st) {
    const rf_plan_host& h = p->h;
    const size_t smem = static_cast<size_t>(h.n_mels) * 33 * 4;
    dim3 grid((T + 31) / 32, B);
    k_inverse_mel<<<grid, 256, smem, st>>>(d_mel, T, h.n_mels, h.n_live, h.F, p->d_thomas, p->d_binrow_ptr,
                                           p->d_binrow_m, p->d_binrow_w, p->d_bins, out_mode, out);
    RF_CUDA_LAUNCH_CHECK("k_inverse_mel");
    return RF_OK;
}

// optional per-kernel-class CUDA-event timing (bench.py's live roofline measurement)
struct gl_prof {
    std::vector<cudaEvent_t> ev[3][2];  // [istft, assemble, stft][begin,end]
    cudaError_t mark(int cls, int end, cudaStream_t st) {
        cudaEvent_t e;
        cudaError_t rc = cudaEventCreate(&e);
        if (rc != cudaSuccess) return rc;
        ev[cls][end].push_back(e);
        return cudaEventRecord(e, st);
    }
};

// Griffin-Lim main loop on a prepared workspace (S and initial angles in R[1]).
// Griffin-Lim on the generic engine: same recurrence and buffer rotation as below, one CTA per frame
static int gl_loop_generic(rf_plan* p, const gl_ws& w, int B, int T, int n_iter, float momentum_in, float* d_wave,
                           cudaStream_t st) {
    const rf_plan_host& h = p->h;
    int rc = gen_smem_attrs(p);
    if (rc) return rc;
    const rf_gen_tab g = make_gen_tab(p);
    const size_t smem = gen_smem(p);
    const int L = h.H * (T - 1);
    const int c0 = h.N / 2 - (h.N - h.W) / 2;
    const float m = static_cast<float>(static_cast<double>(momentum_in) / (1.0 + static_cast<double>(momentum_in)));
    const dim3 grid_f(T, B), grid_a((L + 255) / 256, B);
    for (int it = 0; it <= n_iter; ++it) {
        const rf_c32* cur = it == 0 ? w.R[1] : w.R[(it - 1) & 1];
        const rf_c32* prev = (it >= 2 && m != 0.f) ? w.R[it & 1] : nullptr;
        k_gen_istft<<<grid_f, 256, smem, st>>>(g, w.S, cur, prev, it == 0 ? 0 : 1, m, T, w.part);
        RF_CUDA_LAUNCH_CHECK("k_gen_istft");
        k_gen_ola<<<grid_a, 256, 0, st>>>(w.part, p->d_win2, T, h.H, h.W, c0, L, d_wave);
        RF_CUDA_LAUNCH_CHECK("k_gen_ola");
        if (it == n_iter) break;
        k_gen_stft<<<grid_f, 256, smem, st>>>(g, d_wave, L, T, w.R[it & 1]);
        RF_CUDA_LAUNCH_CHECK("k_gen_stft");
    }
    return RF_OK;
}

static int gl_loop(rf_plan* p, const gl_ws& w, int B, int T, int n_iter, float momentum_in, float* d_wave,
                   cudaStream_t st, gl_prof* prof = nullptr) {
    const rf_plan_host& h = p->h;
    if (h.generic) return gl_loop_generic(p, w, B, T, n_iter, momentum_in, d_wave, st);
    const rf_gl_tables tb = make_tables(p, 10);
    const int L = h.H * (T - 1);
    // momentum = momentum / (1 + momentum)  (TA/functional/functional.py:300), fp32 like python float->tensor op
    const float m = static_cast<float>(static_cast<double>(momentum_in) / (1.0 + static_cast<double>(momentum_in)));
    const bool dec = h.decimate && p->use_decimation && p->d5.bt != nullptr && w.xd != nullptr;
    const rf_gl_tables tb2 = dec ? make_tables(p, 5) : tb;
    rf_gl_tables tbo = tb2;        // the other sample parity of the decimated grid (edge chunks): frame t0+1 starts (H-1)/2 later
    tbo.wg_inv = p->d5e_wg_inv;
    tbo.ab_inv = p->d5e_ab_inv;
    tbo.off1 = (h.H - 1) / 2;
    const rf_gl_dec_geom dg = rf_dec_geom(T, RF_CHUNK, h.H, h.W);
    const int PLh = ((RF_CHUNK - 1) * h.H + h.W + 1) / 2;
    const size_t smem_i = 2 * RF_PW * sizeof(rf_c32) + static_cast<size_t>(w.PL) * 4;
    const size_t smem_f = 2 * RF_PW * sizeof(rf_c32) + static_cast<size_t>(RF_PW + h.H) * 4;
#if RF_GL_HALF_MINB >= 3
    const size_t smem_ih = 2 * (RF_PW / 2) * sizeof(rf_c32) + static_cast<size_t>(PLh) * 4;                       // half-rate CTAs
    const size_t smem_fh = 2 * (RF_PW / 2) * sizeof(rf_c32) + 2 * RF_XS_HALF_BYTES + 16;   // two staging buffers + mbarriers
#else       // A/B build: the footprint of the merged launch (2 CTAs per SM)
    const size_t smem_ih = smem_i, smem_fh = smem_f;
#endif
    const dim3 grid_i(w.nchunks * 2, B), grid_f(((T + 1) / 2) * 2, B), grid_a((L + 255) / 256, B);
    k_envelope<<<(L + 255) / 256, 256, 0, st>>>(p->d_win2, T, h.H, h.W, L, w.env);
    RF_CUDA_LAUNCH_CHECK("k_envelope");
    for (int it = 0; it <= n_iter; ++it) {
        const rf_c32* cur;
        const rf_c32* prev = nullptr;
        int mode;
        if (it == 0) {
            cur = w.R[1];
            mode = 0;
        } else {
            cur = w.R[(it - 1) & 1];
            mode = 1;
            if (it >= 2 && m != 0.f) prev = w.R[it & 1];
        }
        const bool last = it == n_iter;
        const bool half = dec && !last;   // the final reconstruction is always full rate
        if (prof) RF_CUDA_TRY(prof->mark(0, 0, st));
        if (half) {
            k_istft_half<<<dim3((w.nchunks + dg.nslots) * 2, B), RF_NT, smem_ih, st>>>(
                tb2, tbo, w.S, cur, prev, mode, m, T, RF_CHUNK, PLh, w.nchunks, dg.c_tail, dg.nslots, w.part, w.part_e);
            RF_CUDA_LAUNCH_CHECK("k_istft_half");
        } else
            k_istft_chunk<<<grid_i, RF_NT, smem_i, st>>>(tb, w.S, cur, prev, mode, m, T, RF_CHUNK, w.PL, w.nchunks,
                                                         w.part);
        RF_CUDA_LAUNCH_CHECK("k_istft_chunk");
        if (prof) {
            RF_CUDA_TRY(prof->mark(0, 1, st));
            RF_CUDA_TRY(prof->mark(1, 0, st));
        }
        if (half)
        {
            k_ola_assemble_dec<<<dim3((dg.nxo + 255) / 256, B), 256, 0, st>>>(w.part, w.env, PLh, w.nchunks, dg.nxo, dg.E, w.xd);
            RF_CUDA_LAUNCH_CHECK("k_ola_assemble_dec");
            k_ola_assemble_strips<<<dim3((2 * dg.E + 255) / 256, B), 256, 0, st>>>(w.part, w.part_e, w.env, T, PLh, w.nchunks,
                                                                                   dg.c_tail, dg.nslots, L, dg.nxo, dg.E, w.xd);
        }
        else
            k_ola_assemble<<<grid_a, 256, 0, st>>>(w.part, w.env, T, RF_CHUNK, w.PL, w.nchunks, h.H, h.W, L, d_wave);
        RF_CUDA_LAUNCH_CHECK("k_ola_assemble");
        if (prof) RF_CUDA_TRY(prof->mark(1, 1, st));
        if (last) break;
        if (prof) RF_CUDA_TRY(prof->mark(2, 0, st));
        if (dec) {
            k_stft_edge<<<dim3(dg.n_edge_pairs * 2, B), RF_NT, smem_f, st>>>(tb, w.xd, L, T, h.H, dg.nxo, dg.E, dg.pr_tail,
                                                                            w.R[it & 1]);
            RF_CUDA_LAUNCH_CHECK("k_stft_edge");
            // the half-rate pairs [3, pr_tail): RF_STFT_HALF_PAIRS consecutive pairs per CTA
            k_stft_half<<<dim3((dg.pr_tail - 3 + RF_STFT_HALF_PAIRS - 1) / RF_STFT_HALF_PAIRS * 2, B), RF_NT, smem_fh, st>>>(
                tb2, w.xd, L, T, h.H, dg.nxo, dg.E, 3, dg.pr_tail, w.R[it & 1]);
            RF_CUDA_LAUNCH_CHECK("k_stft_half");
        } else
            k_stft_pair<<<grid_f, RF_NT, smem_f, st>>>(tb, d_wave, L, T, h.H, w.R[it & 1]);
        RF_CUDA_LAUNCH_CHECK("k_stft_pair");
        if (prof) RF_CUDA_TRY(prof->mark(2, 1, st));
    }
    return RF_OK;
}

static int gl_prepare_angles(rf_plan* p, const gl_ws& w, const void* d_init_angles, int B, int T,
                             cudaStream_t st) {
    const rf_plan_host& h = p->h;
    if (d_init_angles) {
        dim3 grid((h.n_live + 31) / 32, (T + 31) / 32, B), blk(32, 32);
        k_gather_FT_to_TJ<float2><<<grid, blk, 0, st>>>(static_cast<const float2*>(d_init_angles), p->d_bins,
                                                        h.F, T, h.n_live, reinterpret_cast<float2*>(w.R[1]));
        RF_CUDA_LAUNCH_CHECK("k_gather_FT_to_TJ<angles>");
    } else {
        const size_t n = static_cast<size_t>(B) * T * h.n_live;
        k_fill_c32<<<static_cast<unsigned>((n + 255) / 256), 256, 0, st>>>(w.R[1], n, 1.f, 0.f);
        RF_CUDA_LAUNCH_CHECK("k_fill_c32");
    }
    return RF_OK;
}

// Prologue of the Griffin-Lim entry points `who`: argument checks, plan upload, shared-memory limits, workspace layout.
static int gl_setup(rf_plan* p, const float* d_in, float* d_wave, void* d_ws, size_t ws_bytes, int B, int T, int n_iter,
                    float momentum, const char* who, gl_ws* w) {
    if (!p || !d_in || !d_wave || !d_ws || B <= 0 || n_iter < 0)
        return rf_fail(RF_ERR_INVALID, std::string(who) + ": bad argument");
    if (!(momentum >= 0.f && momentum < 1.f))
        return rf_fail(RF_ERR_INVALID, "momentum must be in range [0, 1). Found: " + std::to_string(momentum));
    int rc = check_T(p, T, who);
    if (rc) return rc;
    if ((rc = rf_plan_upload(p))) return rc;
    if ((rc = set_smem_attrs())) return rc;
    *w = gl_layout(p, B, T, d_ws);
    if (ws_bytes < w->total) return rf_fail(RF_ERR_INVALID, std::string(who) + ": workspace too small");
    return RF_OK;
}

extern "C" int rf_griffinlim(rf_plan* p, const float* d_lin, const void* d_init_angles, int B, int T,
                             int n_iter, float momentum, float* d_wave, void* d_ws, size_t ws_bytes,
                             void* stream) {
    gl_ws w;
    int rc = gl_setup(p, d_lin, d_wave, d_ws, ws_bytes, B, T, n_iter, momentum, "rf_griffinlim", &w);
    if (rc) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const rf_plan_host& h = p->h;
    dim3 grid((h.n_live + 31) / 32, (T + 31) / 32, B), blk(32, 32);
    k_gather_FT_to_TJ<float><<<grid, blk, 0, st>>>(d_lin, p->d_bins, h.F, T, h.n_live, w.S);
    RF_CUDA_LAUNCH_CHECK("k_gather_FT_to_TJ<lin>");
    if ((rc = gl_prepare_angles(p, w, d_init_angles, B, T, st))) return rc;
    return gl_loop(p, w, B, T, n_iter, momentum, d_wave, st);
}

// inverse mel + Griffin-Lim; `prof` (optional) receives CUDA events around the loop's kernels
static int mel_to_wave(rf_plan* p, const float* d_mel, const void* d_init_angles, int B, int T, int n_iter,
                       float momentum, float* d_wave, void* d_ws, size_t ws_bytes, cudaStream_t st, const char* who,
                       gl_prof* prof) {
    gl_ws w;
    int rc = gl_setup(p, d_mel, d_wave, d_ws, ws_bytes, B, T, n_iter, momentum, who, &w);
    if (rc) return rc;
    if ((rc = launch_inverse_mel(p, d_mel, B, T, 0, w.S, st))) return rc;
    if ((rc = gl_prepare_angles(p, w, d_init_angles, B, T, st))) return rc;
    return gl_loop(p, w, B, T, n_iter, momentum, d_wave, st, prof);
}

extern "C" int rf_mel_to_wave(rf_plan* p, const float* d_mel, const void* d_init_angles, int B, int T,
                              int n_iter, float momentum, float* d_wave, void* d_ws, size_t ws_bytes,
                              void* stream) {
    return mel_to_wave(p, d_mel, d_init_angles, B, T, n_iter, momentum, d_wave, d_ws, ws_bytes,
                       static_cast<cudaStream_t>(stream), "rf_mel_to_wave", nullptr);
}

// Same as rf_mel_to_wave, with every Griffin-Lim kernel launch bracketed by CUDA events on
// `stream`; synchronises the stream and returns the summed device time per kernel class.
//   ms_out[3]       host: total ms of {k_istft_chunk, k_ola_assemble, k_stft_pair}
//   launches_out[3] host: launches per class
extern "C" int rf_mel_to_wave_profiled(rf_plan* p, const float* d_mel, const void* d_init_angles, int B, int T,
                                       int n_iter, float momentum, float* d_wave, void* d_ws, size_t ws_bytes,
                                       void* stream, float* ms_out, int* launches_out) {
    if (!ms_out || !launches_out) return rf_fail(RF_ERR_INVALID, "rf_mel_to_wave_profiled: bad argument");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    gl_prof prof;
    const int rc = mel_to_wave(p, d_mel, d_init_angles, B, T, n_iter, momentum, d_wave, d_ws, ws_bytes, st,
                               "rf_mel_to_wave_profiled", &prof);
    cudaError_t e = cudaStreamSynchronize(st);
    for (int c = 0; c < 3; ++c) {
        ms_out[c] = 0.f;
        launches_out[c] = static_cast<int>(prof.ev[c][1].size());
        for (size_t i = 0; i < prof.ev[c][1].size() && i < prof.ev[c][0].size(); ++i) {
            float ms = 0.f;
            if (rc == RF_OK && e == cudaSuccess && cudaEventElapsedTime(&ms, prof.ev[c][0][i], prof.ev[c][1][i]) == cudaSuccess)
                ms_out[c] += ms;
        }
        for (int k = 0; k < 2; ++k)
            for (cudaEvent_t ev : prof.ev[c][k]) cudaEventDestroy(ev);
    }
    if (rc) return rc;
    if (e != cudaSuccess) return rf_fail(RF_ERR_CUDA, std::string("cudaStreamSynchronize: ") + cudaGetErrorString(e));
    return RF_OK;
}

// ---- periodic Griffin-Lim (seamless loops): frames [B][T][W] of the generic engine, waveform [B][T * hop] -------------
struct per_ws {
    float* S;
    rf_c32* R[2];
    float* frames;
    size_t total;
};

static per_ws per_layout(const rf_plan* p, int B, int T, void* base) {
    per_ws w;
    const size_t bt = static_cast<size_t>(B) * T * p->h.n_live;
    unsigned char* b = static_cast<unsigned char*>(base);
    size_t off = 0;
    w.S = reinterpret_cast<float*>(b + off);
    off += align256(bt * 4);
    w.R[0] = reinterpret_cast<rf_c32*>(b + off);
    off += align256(bt * 8);
    w.R[1] = reinterpret_cast<rf_c32*>(b + off);
    off += align256(bt * 8);
    w.frames = reinterpret_cast<float*>(b + off);
    off += align256(static_cast<size_t>(B) * T * p->h.W * 4);
    w.total = off;
    return w;
}

extern "C" size_t rf_mel_to_wave_periodic_workspace_bytes(const rf_plan* p, int B, int T) {
    if (!p || B <= 0 || T <= 0) return 0;
    return per_layout(p, B, T, nullptr).total;
}

extern "C" int rf_mel_to_wave_periodic(rf_plan* p, const float* d_mel, const void* d_init_angles, int B, int T, int n_iter,
                                       float momentum, float* d_wave, void* d_ws, size_t ws_bytes, void* stream) {
    const char* who = "rf_mel_to_wave_periodic";
    if (!p || !d_mel || !d_wave || !d_ws || B <= 0 || T <= 0 || n_iter < 0)
        return rf_fail(RF_ERR_INVALID, std::string(who) + ": bad argument");
    if (!(momentum >= 0.f && momentum < 1.f))
        return rf_fail(RF_ERR_INVALID, "momentum must be in range [0, 1). Found: " + std::to_string(momentum));
    const rf_plan_host& h = p->h;
    if (!h.mixed_radix)
        return rf_fail(RF_ERR_UNSUPPORTED, std::string(who) + ": n_fft / 2 must be 2^a 3^b 5^c 7^d <= 14000");
    if (h.H > h.W)
        return rf_fail(RF_ERR_INVALID, std::string(who) + ": hop_length > win_length leaves samples no frame covers");
    if (static_cast<long>(T) * h.H > INT32_MAX / 2) return rf_fail(RF_ERR_INVALID, std::string(who) + ": too many frames");
    int rc = rf_plan_upload(p);
    if (rc) return rc;
    if ((rc = set_smem_attrs())) return rc;
    if ((rc = gen_smem_attrs(p))) return rc;
    static rf_dev_once once;
    RF_CUDA_TRY(rf_set_smem_once(once, k_per_stft, 227 * 1024));
    const per_ws w = per_layout(p, B, T, d_ws);
    if (ws_bytes < w.total) return rf_fail(RF_ERR_INVALID, std::string(who) + ": workspace too small");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if ((rc = launch_inverse_mel(p, d_mel, B, T, 0, w.S, st))) return rc;
    gl_ws gw{};                     // gl_prepare_angles writes the initial angles to R[1]
    gw.R[1] = w.R[1];
    if ((rc = gl_prepare_angles(p, gw, d_init_angles, B, T, st))) return rc;
    const rf_gen_tab g = make_gen_tab(p);
    const size_t smem = gen_smem(p);
    const int L = h.H * T;
    const int c0 = h.N / 2 - (h.N - h.W) / 2;
    // the recurrence and buffer rotation of gl_loop / gl_loop_generic (TA/functional/functional.py:300-340)
    const float m = static_cast<float>(static_cast<double>(momentum) / (1.0 + static_cast<double>(momentum)));
    const dim3 grid_f(T, B), grid_a((L + 255) / 256, B);
    for (int it = 0; it <= n_iter; ++it) {
        const rf_c32* cur = it == 0 ? w.R[1] : w.R[(it - 1) & 1];
        const rf_c32* prev = (it >= 2 && m != 0.f) ? w.R[it & 1] : nullptr;
        k_gen_istft<<<grid_f, 256, smem, st>>>(g, w.S, cur, prev, it == 0 ? 0 : 1, m, T, w.frames);
        RF_CUDA_LAUNCH_CHECK("k_gen_istft");
        k_per_ola<<<grid_a, 256, 0, st>>>(w.frames, p->d_win2, T, h.H, h.W, c0, L, d_wave);
        RF_CUDA_LAUNCH_CHECK("k_per_ola");
        if (it == n_iter) break;
        k_per_stft<<<grid_f, 256, smem, st>>>(g, d_wave, L, T, w.R[it & 1]);
        RF_CUDA_LAUNCH_CHECK("k_per_stft");
    }
    return RF_OK;
}

extern "C" int rf_inverse_mel(rf_plan* p, const float* d_mel, int B, int T, float* d_lin, void* stream) {
    if (!p || !d_mel || !d_lin || B <= 0 || T <= 0) return rf_fail(RF_ERR_INVALID, "rf_inverse_mel: bad argument");
    int rc = rf_plan_upload(p);
    if (rc) return rc;
    if ((rc = set_smem_attrs())) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    RF_CUDA_TRY(cudaMemsetAsync(d_lin, 0, static_cast<size_t>(B) * p->h.F * T * 4, st));
    return launch_inverse_mel(p, d_mel, B, T, 1, d_lin, st);
}

static int check_L(const rf_plan* p, int L, const char* who) {
    if (L <= p->h.N / 2)
        return rf_fail(RF_ERR_INVALID,
                       std::string(who) + ": Padding size should be less than the corresponding input "
                       "dimension (L = " + std::to_string(L) + " must exceed n_fft/2 = " +
                           std::to_string(p->h.N / 2) + ")");
    return RF_OK;
}

extern "C" int rf_stft_mel(rf_plan* p, const float* d_wave, int B, int L, float* d_mel, void* stream) {
    if (!p || !d_wave || !d_mel || B <= 0) return rf_fail(RF_ERR_INVALID, "rf_stft_mel: bad argument");
    int rc = check_L(p, L, "rf_stft_mel");
    if (rc) return rc;
    if ((rc = rf_plan_upload(p))) return rc;
    if ((rc = set_smem_attrs())) return rc;
    const rf_plan_host& h = p->h;
    const int T = 1 + L / h.H;
    if (h.generic) {
        if ((rc = gen_smem_attrs(p))) return rc;
        cudaStream_t st = static_cast<cudaStream_t>(stream);
        rf_c32* tmp = nullptr;
        RF_CUDA_TRY(cudaMallocAsync(reinterpret_cast<void**>(&tmp), static_cast<size_t>(B) * T * h.n_live * 8, st));
        k_gen_stft<<<dim3(T, B), 256, gen_smem(p), st>>>(make_gen_tab(p), d_wave, L, T, tmp);
        RF_CUDA_LAUNCH_CHECK("k_gen_stft");
        k_gen_mel_from_TJ<<<dim3((T + 127) / 128, h.n_mels, B), 128, 0, st>>>(tmp, T, h.n_live, h.n_mels, p->d_melcol_ptr,
                                                                             p->d_melcol_j, p->d_melcol_w, d_mel);
        RF_CUDA_LAUNCH_CHECK("k_gen_mel_from_TJ");
        RF_CUDA_TRY(cudaFreeAsync(tmp, st));
        return RF_OK;
    }
    const size_t xs_n = (RF_PW + h.H) + ((RF_PW + h.H) & 1);
    const size_t smem = 2 * RF_PW * sizeof(rf_c32) + xs_n * 4 + 2 * static_cast<size_t>(h.n_live) * 8;
    if (smem > 227 * 1024) return rf_fail(RF_ERR_UNSUPPORTED, "rf_stft_mel: live band too wide for the fused kernel");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    dim3 grid((T + 1) / 2, B);
    k_stft_mel_pair<<<grid, RF_NT, smem, st>>>(make_tables(p), d_wave, L, T, h.n_mels, p->d_melcol_ptr,
                                               p->d_melcol_j, p->d_melcol_w, d_mel);
    RF_CUDA_LAUNCH_CHECK("k_stft_mel_pair");
    return RF_OK;
}

extern "C" int rf_stft(rf_plan* p, const float* d_wave, int B, int L, void* d_spec, void* stream) {
    if (!p || !d_wave || !d_spec || B <= 0) return rf_fail(RF_ERR_INVALID, "rf_stft: bad argument");
    int rc = check_L(p, L, "rf_stft");
    if (rc) return rc;
    if ((rc = rf_plan_upload(p))) return rc;
    if ((rc = set_smem_attrs())) return rc;
    const rf_plan_host& h = p->h;
    const int T = 1 + L / h.H;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    rf_c32* tmp = nullptr;
    const size_t n = static_cast<size_t>(B) * T * h.n_live;
    RF_CUDA_TRY(cudaMallocAsync(reinterpret_cast<void**>(&tmp), n * 8, st));
    if (h.generic) {
        if ((rc = gen_smem_attrs(p))) return rc;
        k_gen_stft<<<dim3(T, B), 256, gen_smem(p), st>>>(make_gen_tab(p), d_wave, L, T, tmp);
        RF_CUDA_LAUNCH_CHECK("k_gen_stft");
    } else {
        const size_t smem_f = 2 * RF_PW * sizeof(rf_c32) + static_cast<size_t>(RF_PW + h.H) * 4;
        dim3 grid_f(((T + 1) / 2) * 2, B);
        k_stft_pair<<<grid_f, RF_NT, smem_f, st>>>(make_tables(p), d_wave, L, T, h.H, tmp);
        RF_CUDA_LAUNCH_CHECK("k_stft_pair");
    }
    RF_CUDA_TRY(cudaMemsetAsync(d_spec, 0, static_cast<size_t>(B) * h.F * T * 8, st));
    dim3 grid((h.n_live + 31) / 32, (T + 31) / 32, B), blk(32, 32);
    k_scatter_TJ_to_FT<float2><<<grid, blk, 0, st>>>(reinterpret_cast<const float2*>(tmp), p->d_bins, h.F, T,
                                                     h.n_live, static_cast<float2*>(d_spec));
    RF_CUDA_LAUNCH_CHECK("k_scatter_TJ_to_FT");
    RF_CUDA_TRY(cudaFreeAsync(tmp, st));
    return RF_OK;
}

extern "C" int rf_mel_scale(rf_plan* p, const float* d_spec, int B, int T, float* d_mel, void* stream) {
    if (!p || !d_spec || !d_mel || B <= 0 || T <= 0) return rf_fail(RF_ERR_INVALID, "rf_mel_scale: bad argument");
    int rc = rf_plan_upload(p);
    if (rc) return rc;
    const rf_plan_host& h = p->h;
    dim3 grid((T + 127) / 128, h.n_mels, B);
    k_mel_scale<<<grid, 128, 0, static_cast<cudaStream_t>(stream)>>>(d_spec, h.F, T, h.n_mels, p->d_melcol_ptr,
                                                                   p->d_melcol_j, p->d_melcol_w, p->d_bins, d_mel);
    RF_CUDA_LAUNCH_CHECK("k_mel_scale");
    return RF_OK;
}

extern "C" int rf_image_to_mel(const uint8_t* d_img, int height, int width, int stereo, float power,
                               float max_value, float* d_mel, void* stream) {
    if (!d_img || !d_mel || height <= 0 || width <= 0 || !(power > 0.f))
        return rf_fail(RF_ERR_INVALID, "rf_image_to_mel: bad argument");
    dim3 grid((width + 127) / 128, height, stereo ? 2 : 1);
    // np.power(data, 1 / power): the exponent is a python float (fp64) cast to the array dtype
    const float inv_power = static_cast<float>(1.0 / static_cast<double>(power));
    k_image_to_mel<<<grid, 128, 0, static_cast<cudaStream_t>(stream)>>>(d_img, height, width, stereo, inv_power,
                                                                      max_value, d_mel);
    RF_CUDA_LAUNCH_CHECK("k_image_to_mel");
    return RF_OK;
}

extern "C" int rf_mel_to_image(const float* d_mel, int channels, int height, int width, float power,
                               uint8_t* d_img, float* d_max, void* stream) {
    if (!d_mel || !d_img || !d_max || height <= 0 || width <= 0)
        return rf_fail(RF_ERR_INVALID, "rf_mel_to_image: bad argument");
    if (channels != 1 && channels != 2)
        return rf_fail(RF_ERR_INVALID, "Unsupported number of channels: " + std::to_string(channels));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    RF_CUDA_TRY(cudaMemsetAsync(d_max, 0, 4, st));
    const size_t n = static_cast<size_t>(channels) * height * width;
    k_absmax<<<2 * rf_num_sms(), 256, 0, st>>>(d_mel, n, 0, d_max);
    RF_CUDA_LAUNCH_CHECK("k_absmax");
    dim3 grid((width + 127) / 128, height);
    k_mel_to_image<<<grid, 128, 0, st>>>(d_mel, channels, height, width, power, d_max, d_img);
    RF_CUDA_LAUNCH_CHECK("k_mel_to_image");
    return RF_OK;
}

extern "C" int rf_wave_to_int16(const float* d_wave, int channels, int L, int normalize, int16_t* d_pcm,
                                float* d_scratch, void* stream) {
    if (!d_wave || !d_pcm || !d_scratch || channels <= 0 || L <= 0)
        return rf_fail(RF_ERR_INVALID, "rf_wave_to_int16: bad argument");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (normalize) {
        RF_CUDA_TRY(cudaMemsetAsync(d_scratch, 0, 4, st));
        k_absmax<<<2 * rf_num_sms(), 256, 0, st>>>(d_wave, static_cast<size_t>(channels) * L, 1, d_scratch);
        RF_CUDA_LAUNCH_CHECK("k_absmax");
    }
    k_wave_to_int16<<<(L + 255) / 256, 256, 0, st>>>(d_wave, channels, L, d_scratch, normalize, d_pcm);
    RF_CUDA_LAUNCH_CHECK("k_wave_to_int16");
    return RF_OK;
}
