// Host plan builder for path (a).  See rf_plan.h.
//
// Reference arithmetic restated here (for table construction only):
//   window        torch.hann_window(win, periodic)    TA/transforms/_transforms.py:94
//   mel fbanks    melscale_fbanks / _create_triangular_filterbank
//                                                      TA/functional/functional.py:488-587
//   inverse mel   relu(lstsq(fb^T, mel, "gels"))       TA/transforms/_transforms.py:508
//                 == relu(fb (fb^T fb)^{-1} mel) (minimum-norm solution; fb^T fb is
//                 tridiagonal because only neighbouring triangles overlap)
#include "rf_plan.h"

#include <algorithm>
#include <cmath>
#include <cstring>

namespace {

// torch.linspace(start, end, steps) in fp32 (ATen RangeFactories: symmetric evaluation)
std::vector<float> linspace_f32(float start, float end, int steps) {
    std::vector<float> v(steps);
    if (steps == 1) {
        v[0] = start;
        return v;
    }
    const float step = (end - start) / static_cast<float>(steps - 1);
    const int half = steps / 2;
    for (int i = 0; i < steps; ++i) {
        if (i < half)
            v[i] = start + step * static_cast<float>(i);
        else
            v[i] = end - step * static_cast<float>(steps - 1 - i);
    }
    return v;
}

double hz_to_mel(double f, bool slaney) {
    if (!slaney) return 2595.0 * std::log10(1.0 + f / 700.0);
    const double f_sp = 200.0 / 3.0, min_log_hz = 1000.0;
    const double min_log_mel = min_log_hz / f_sp, logstep = std::log(6.4) / 27.0;
    if (f >= min_log_hz) return min_log_mel + std::log(f / min_log_hz) / logstep;
    return f / f_sp;
}

// follows the fp32 op sequence of torchaudio (pow/log rounding may differ by 1 ulp from
// torch's vectorised math; pass `fb` from Python for bit parity)
std::vector<float> melscale_fbanks_f32(int n_freqs, float f_min, float f_max, int n_mels,
                                       int sample_rate, bool norm_slaney, bool scale_slaney) {
    std::vector<float> all_freqs = linspace_f32(0.0f, static_cast<float>(sample_rate / 2), n_freqs);
    const float m_min = static_cast<float>(hz_to_mel(f_min, scale_slaney));
    const float m_max = static_cast<float>(hz_to_mel(f_max, scale_slaney));
    std::vector<float> m_pts = linspace_f32(m_min, m_max, n_mels + 2);
    std::vector<float> f_pts(n_mels + 2);
    for (int i = 0; i < n_mels + 2; ++i) {
        if (!scale_slaney) {
            float e = m_pts[i] / 2595.0f;
            f_pts[i] = 700.0f * (std::pow(10.0f, e) - 1.0f);
        } else {
            const float f_sp = 200.0f / 3.0f, min_log_hz = 1000.0f;
            const float min_log_mel = min_log_hz / f_sp;
            const float logstep = static_cast<float>(std::log(6.4) / 27.0);
            float f = f_sp * m_pts[i];
            if (m_pts[i] >= min_log_mel) f = min_log_hz * std::exp(logstep * (m_pts[i] - min_log_mel));
            f_pts[i] = f;
        }
    }
    std::vector<float> fb(static_cast<size_t>(n_freqs) * n_mels);
    for (int k = 0; k < n_freqs; ++k) {
        for (int m = 0; m < n_mels; ++m) {
            const float fd0 = f_pts[m + 1] - f_pts[m];
            const float fd1 = f_pts[m + 2] - f_pts[m + 1];
            const float down = (-1.0f * (f_pts[m] - all_freqs[k])) / fd0;
            const float up = (f_pts[m + 2] - all_freqs[k]) / fd1;
            float v = std::max(0.0f, std::min(down, up));
            if (norm_slaney) v *= 2.0f / (f_pts[m + 2] - f_pts[m]);
            fb[static_cast<size_t>(k) * n_mels + m] = v;
        }
    }
    return fb;
}

#include "rf_pass_b_perm.inc"

// kernel-side forms of the per-bin / per-sample tables (rf_bin_tabs) for one prime-factor grid
// swap (NA = 5, inverse tables only): the OTHER sample parity of the decimated grid — frame t0 takes the odd live samples
// n' = 2u+1 (so it, not frame t0+1, carries the extra modulation exp(2 pi i k/N)) and frame t0+1 the even ones: the
// half-rate inverse transform then yields the waveform samples the regular half-rate pass skips (rf_plan_host::t5e)
void build_bin_tabs(const rf_plan_host& p, int NA, const std::vector<uint32_t>& pp, const std::vector<float>* ph_odd,
                    rf_bin_tabs& t, bool swap = false) {
    const int W = NA * 441;
    const int J = p.n_live;
    t.bt.resize(J);
    t.ab_inv.resize(static_cast<size_t>(J) * 4);
    t.ab_fwd.resize(static_cast<size_t>(J) * 4);
    std::vector<char> hit[2] = {std::vector<char>(2 * W, 0), std::vector<char>(2 * W, 0)};
    for (int j = 0; j < J; ++j) {
        const uint32_t q = pp[j];
        const int r = q & 3, idx = (q >> 2) & 8191, idx2 = (q >> 15) & 8191, k7 = q >> 28;
        const int rp = (4 - r) & 3;
        const int off = (r >> 1) * W + idx, off2 = (rp >> 1) * W + idx2;
        const bool self = idx2 == idx && rp == r;
        t.bt[j] = static_cast<uint32_t>(off) | (static_cast<uint32_t>(off2) << 14) | (self ? 1u << 31 : 0u);
        const int g = j < p.n_even ? 0 : 1;
        hit[g][off] = hit[g][off2] = 1;
        // ph = exp(-2 pi i 3k/8) (frame offset (N-W)/2 = 3N/8), po = exp(-2 pi i k/N) (odd-sample frame, NA = 5 only)
        const double a_ph = -2.0 * M_PI * ((3 * k7) & 7) / 8.0;
        const double phx = std::cos(a_ph), phy = std::sin(a_ph);
        double pox = 1.0, poy = 0.0;
        if (ph_odd) {
            const double a_po = -2.0 * M_PI * static_cast<double>(p.bins[j]) / p.N;
            pox = std::cos(a_po);
            poy = std::sin(a_po);
        }
        // e = ph * po
        const double ex = phx * pox - phy * poy, ey = phx * poy + phy * pox;
        float* ai = &t.ab_inv[static_cast<size_t>(j) * 4];
        if (!swap) {
            ai[0] = static_cast<float>(phx);      // alpha = conj(ph)
            ai[1] = static_cast<float>(-phy);
            ai[2] = static_cast<float>(ey);       // beta = i conj(e) = (ey, ex)
            ai[3] = static_cast<float>(ex);
        } else {
            ai[0] = static_cast<float>(ex);       // alpha = conj(ph) conj(po) = conj(e)
            ai[1] = static_cast<float>(-ey);
            ai[2] = static_cast<float>(phy);      // beta = i conj(ph) = (phy, phx)
            ai[3] = static_cast<float>(phx);
        }
        float* af = &t.ab_fwd[static_cast<size_t>(j) * 4];
        af[0] = static_cast<float>(0.5 * phx);   // gamma = ph / 2
        af[1] = static_cast<float>(0.5 * phy);
        af[2] = static_cast<float>(0.5 * ey);    // delta = -i e / 2 = (ey, -ex) / 2
        af[3] = static_cast<float>(-0.5 * ex);
    }
    t.zpos.clear();
    for (int g = 0; g < 2; ++g) {
        t.nz[g] = 0;
        for (int i = 0; i < 2 * W; ++i)
            if (!hit[g][i]) {
                t.zpos.push_back(static_cast<uint16_t>(i));
                ++t.nz[g];
            }
    }
    // radix-9 pass: item (a, c) of slot tau, and per (b, slot) the two windows and the r = 1 modulation at that sample
    const uint16_t* perm = rf_pass_b_perm(NA);
    const int n_items = 49 * NA;
    t.items.resize(n_items);
    t.wg_fwd.assign(static_cast<size_t>(W) * 4, 0.f);
    t.wg_inv.assign(static_cast<size_t>(W) * 4, 0.f);
    for (int tau = 0; tau < n_items; ++tau) {
        const int a = perm[tau] / 49, c = perm[tau] % 49;
        const int base = (441 * a + (W / 49) * c) % W;
        t.items[tau] = static_cast<uint32_t>(a * 441 + c) | (static_cast<uint32_t>(base) << 12);
        for (int bq = 0; bq < 9; ++bq) {
            const int u = (base + (W / 9) * bq) % W;            // sample index within the (decimated) frame
            const double ang = 2.0 * M_PI * static_cast<double>(u) / (NA == 5 ? p.N / 2 : p.N);
            const double w0 = NA == 5 ? p.window[2 * u + (swap ? 1 : 0)] : p.window[u];
            const double w1 = NA == 5 ? p.window[2 * u + (swap ? 0 : 1)] : p.window[u];
            const double fs = NA == 5 ? 2.0 : 1.0;              // half the samples carry the same spectrum at half the level
            const size_t o = (static_cast<size_t>(bq) * n_items + tau) * 4;
            t.wg_fwd[o] = static_cast<float>(fs * w0);
            t.wg_fwd[o + 1] = static_cast<float>(fs * w1);
            t.wg_fwd[o + 2] = static_cast<float>(std::cos(ang));
            t.wg_fwd[o + 3] = static_cast<float>(-std::sin(ang));
            t.wg_inv[o] = static_cast<float>(w0 / p.N);
            t.wg_inv[o + 1] = static_cast<float>(w1 / p.N);
            t.wg_inv[o + 2] = static_cast<float>(std::cos(ang));
            t.wg_inv[o + 3] = static_cast<float>(std::sin(ang));
        }
    }
}

}  // namespace

std::string rf_plan_build_host(const rf_plan_desc& d, const float* window, const float* fb_in,
                               rf_plan_host& p, int& code) {
    code = RF_ERR_INVALID;
    if (d.n_fft <= 0 || d.win_length <= 0 || d.hop_length <= 0 || d.n_mels <= 0 || d.sample_rate <= 0)
        return "rf_plan_create: non-positive geometry";
    if (d.win_length > d.n_fft) return "rf_plan_create: win_length > n_fft";
    if (d.f_min > d.f_max) return "Require f_min <= f_max";  // TA/transforms/_transforms.py:473
    code = RF_ERR_UNSUPPORTED;
    // 44.1 kHz defaults (win 4410 = 10*9*49, n_fft 17640, hop | win): the prime-factor engine.  Anything else (other sample
    // rates: 48 kHz -> 4800 / 19200 / 480, 22.05 kHz -> 2205 / 8820 / 220 where hop does not divide win, custom window or
    // padding durations) runs on the generic mixed-radix engine.
    p.generic = d.win_length != RF_W || d.n_fft != RF_N || d.hop_length > RF_W || (RF_W % d.hop_length) != 0;
    if (p.generic) {
        if (d.n_fft & 1) return "rf_plan_create: n_fft must be even (generic FFT engine packs two real samples per point)";
        if (d.n_fft / 2 > 14000)
            return "rf_plan_create: n_fft = " + std::to_string(d.n_fft) + " exceeds the generic engine's shared-memory frame "
                   "(n_fft <= 28000, i.e. sample rates up to 70 kHz with the default 400 ms padding)";
    }
    // the generic engine's radices, also those of the periodic (loop) Griffin-Lim on every plan: the prime-factor geometry's
    // n_fft / 2 = 8820 = 4 * 3 * 3 * 5 * 7 * 7 always factors
    {
        int n2 = d.n_fft / 2;
        p.radices.clear();
        const int cand[5] = {4, 2, 3, 5, 7};
        for (int r : cand)
            while (n2 > 0 && n2 % r == 0 && !(r == 2 && n2 % 4 == 0)) {
                p.radices.push_back(r);
                n2 /= r;
            }
        if (p.generic && n2 != 1)
            return "rf_plan_create: n_fft/2 = " + std::to_string(d.n_fft / 2) + " has a prime factor > 7; the generic FFT engine "
                   "handles 2^a 3^b 5^c 7^d";
        if (p.generic && p.radices.size() > 16) return "rf_plan_create: too many FFT stages";
        p.mixed_radix = n2 == 1 && p.radices.size() <= 16 && (d.n_fft % 2) == 0 && d.n_fft / 2 <= 14000;
    }
    p.d = d;
    p.N = d.n_fft;
    p.W = d.win_length;
    p.H = d.hop_length;
    p.F = d.n_fft / 2 + 1;
    p.n_mels = d.n_mels;

    // ---- window
    p.window.resize(p.W);
    for (int n = 0; n < p.W; ++n)
        p.window[n] = window ? window[n]
                             : static_cast<float>(0.5 - 0.5 * std::cos(2.0 * M_PI * n / p.W));

    // ---- filterbank
    if (fb_in)
        p.fb.assign(fb_in, fb_in + static_cast<size_t>(p.F) * p.n_mels);
    else
        p.fb = melscale_fbanks_f32(p.F, d.f_min, d.f_max, p.n_mels, d.sample_rate,
                                   d.mel_norm_slaney != 0, d.mel_scale_slaney != 0);

    // ---- live bins and private order: (even k | odd k), then r = k%4, then PFA position of k/4
    struct Ent {
        int k, r, idx;
    };
    std::vector<Ent> ents;
    p.fb_nnz = 0;
    for (int k = 0; k < p.F; ++k) {
        bool live = d.full_band != 0;
        for (int m = 0; m < p.n_mels; ++m)
            if (p.fb[static_cast<size_t>(k) * p.n_mels + m] != 0.0f) {
                live = true;
                ++p.fb_nnz;
            }
        if (!live) continue;
        const int mm = k >> 2;
        ents.push_back({k, k & 3, rf_pfa_spec_pos(mm % RF_NA, mm % RF_NB, mm % RF_NC)});
    }
    if (ents.empty()) {
        code = RF_ERR_INVALID;
        return "rf_plan_create: mel filterbank is identically zero";
    }
    if (!p.generic) std::sort(ents.begin(), ents.end(), [](const Ent& x, const Ent& y) {
        const int gx = x.k & 1, gy = y.k & 1;
        if (gx != gy) return gx < gy;
        if (x.r != y.r) return x.r < y.r;
        return x.idx < y.idx;
    });
    // Within each r block, interleave the positions round-robin over (idx mod 16) so that any 16
    // consecutive bins (a half warp of 8-byte shared-memory accesses at V[idx] and at the partner
    // position 4409-idx) fall in 16 distinct bank pairs.
    if (!p.generic) {
        std::vector<Ent> out;
        out.reserve(ents.size());
        size_t i0 = 0;
        while (i0 < ents.size()) {
            size_t i1 = i0;
            while (i1 < ents.size() && ents[i1].r == ents[i0].r && ((ents[i1].k ^ ents[i0].k) & 1) == 0) ++i1;
            std::vector<std::vector<Ent>> cls(16);
            for (size_t i = i0; i < i1; ++i) cls[ents[i].idx & 15].push_back(ents[i]);
            std::vector<size_t> cur(16, 0);
            size_t left = i1 - i0;
            while (left) {
                for (int c = 0; c < 16; ++c)
                    if (cur[c] < cls[c].size()) {
                        out.push_back(cls[c][cur[c]++]);
                        --left;
                    }
            }
            i0 = i1;
        }
        ents.swap(out);
    }
    p.n_live = static_cast<int>(ents.size());
    p.bins.resize(p.n_live);
    p.pp.resize(p.n_live);
    p.jofk.assign(p.F, -1);
    p.n_even = 0;
    p.k_lo = p.F;
    p.k_hi = -1;
    for (int j = 0; j < p.n_live; ++j) {
        const int k = ents[j].k;
        p.bins[j] = k;
        p.jofk[k] = j;
        if ((k & 1) == 0) ++p.n_even;
        p.k_lo = std::min(p.k_lo, k);
        p.k_hi = std::max(p.k_hi, k);
        const int kp = (p.N - k) % p.N;
        const int mp = kp >> 2;
        const uint32_t idx2 = rf_pfa_spec_pos(mp % RF_NA, mp % RF_NB, mp % RF_NC);
        p.pp[j] = static_cast<uint32_t>(ents[j].r) | (static_cast<uint32_t>(ents[j].idx) << 2) |
                  (idx2 << 15) | (static_cast<uint32_t>(k & 7) << 28);
    }

    if (p.mixed_radix) {
        const int N2 = p.N / 2;
        p.roots2.resize(static_cast<size_t>(N2) * 2);
        for (int n = 0; n < N2; ++n) {
            const double ang = -2.0 * M_PI * static_cast<double>(n) / N2;
            p.roots2[2 * n] = static_cast<float>(std::cos(ang));
            p.roots2[2 * n + 1] = static_cast<float>(std::sin(ang));
        }
        p.rootsN.resize(static_cast<size_t>(N2 + 1) * 2);
        for (int k = 0; k <= N2; ++k) {
            const double ang = -2.0 * M_PI * static_cast<double>(k) / p.N;
            p.rootsN[2 * k] = static_cast<float>(std::cos(ang));
            p.rootsN[2 * k + 1] = static_cast<float>(std::sin(ang));
        }
    }
    // ---- modulation x window tables, time-side (Ruritanian) index n'(a,b,c), stored [r][b][c][a]
    if (!p.generic) {
    p.wt_fwd.assign(static_cast<size_t>(4) * p.W * 2, 0.f);
    p.wt_inv.assign(static_cast<size_t>(4) * p.W * 2, 0.f);
    for (int r = 0; r < 4; ++r)
        for (int a = 0; a < RF_NA; ++a)
            for (int b = 0; b < RF_NB; ++b)
                for (int c = 0; c < RF_NC; ++c) {
                    const int n = rf_pfa_n_of(a, b, c);
                    const int pos = b * 490 + c * 10 + a;  // table order [b][c][a]: lanes run over a
                    const long q = (static_cast<long>(r) * n) % p.N;
                    const double ang = -2.0 * M_PI * static_cast<double>(q) / p.N;
                    const double w = p.window[n];
                    const size_t o = (static_cast<size_t>(r) * p.W + pos) * 2;
                    p.wt_fwd[o] = static_cast<float>(w * std::cos(ang));
                    p.wt_fwd[o + 1] = static_cast<float>(w * std::sin(ang));
                    p.wt_inv[o] = static_cast<float>(w * std::cos(ang) / p.N);
                    p.wt_inv[o + 1] = static_cast<float>(-w * std::sin(ang) / p.N);
                }
    }

    // ---- time-decimated loop tables.  Eligible when every live bin k satisfies 2k + 800 <= N/2: the spectrum of a
    // windowed frame at distance >= 800 bins from its content is < 4e-8 of the peak (Hann side lobes fall with the
    // cube of the offset), below fp32 rounding, so sampling the loop signal at every second sample aliases nothing
    // measurable.  Needs an odd hop (frame parities alternate) and an even chunk size.  The full-rate edge strips of the
    // hybrid loop (rf_dec_geom: 3 head pairs, E = W + H, tail chunks from (T-17)/G) are laid out for hop = W/10 = 441,
    // the reference's default step; other odd hops (2205) run the full-rate loop.
    p.decimate = !p.generic && (p.H == 441) && (RF_CHUNK % 2 == 0) && (2 * p.k_hi + 800 <= p.N / 2) && (p.W == 4410);
    if (p.decimate) {
        const int W2 = 2205, N2 = p.N / 2;
        p.pp2.resize(p.n_live);
        p.ph_odd.resize(static_cast<size_t>(p.n_live) * 2);
        for (int j = 0; j < p.n_live; ++j) {
            const int k = p.bins[j];
            const int m = k >> 2;
            const uint32_t idx = rf_pfa_spec_pos(m % 5, m % RF_NB, m % RF_NC);
            const int kp = (N2 - k) % N2;
            const int mp = kp >> 2;
            const uint32_t idx2 = rf_pfa_spec_pos(mp % 5, mp % RF_NB, mp % RF_NC);
            p.pp2[j] = static_cast<uint32_t>(k & 3) | (idx << 2) | (idx2 << 15) | (static_cast<uint32_t>(k & 7) << 28);
            const double ang = -2.0 * M_PI * static_cast<double>(k) / p.N;
            p.ph_odd[2 * j] = static_cast<float>(std::cos(ang));
            p.ph_odd[2 * j + 1] = static_cast<float>(std::sin(ang));
        }
        p.wt2_fwd.assign(static_cast<size_t>(2) * 4 * W2 * 2, 0.f);
        p.wt2_inv.assign(static_cast<size_t>(2) * 4 * W2 * 2, 0.f);
        for (int par = 0; par < 2; ++par)
            for (int r = 0; r < 4; ++r)
                for (int a = 0; a < 5; ++a)
                    for (int b = 0; b < RF_NB; ++b)
                        for (int c = 0; c < RF_NC; ++c) {
                            const int u = rf_pfa2_u_of(a, b, c);
                            const int pos = b * 245 + c * 5 + a;
                            const long q = (static_cast<long>(r) * u) % N2;
                            const double ang = -2.0 * M_PI * static_cast<double>(q) / N2;
                            const double w = p.window[2 * u + par];
                            const size_t o = ((static_cast<size_t>(par) * 4 + r) * W2 + pos) * 2;
                            p.wt2_fwd[o] = static_cast<float>(2.0 * w * std::cos(ang));
                            p.wt2_fwd[o + 1] = static_cast<float>(2.0 * w * std::sin(ang));
                            p.wt2_inv[o] = static_cast<float>(w * std::cos(ang) / p.N);
                            p.wt2_inv[o + 1] = static_cast<float>(-w * std::sin(ang) / p.N);
                        }
    }

    if (!p.generic) build_bin_tabs(p, 10, p.pp, nullptr, p.t10);
    if (p.decimate) {
        build_bin_tabs(p, 5, p.pp2, &p.ph_odd, p.t5);
        build_bin_tabs(p, 5, p.pp2, &p.ph_odd, p.t5e, true);
    }

    // ---- sparse filterbank
    p.melcol_ptr.assign(p.n_mels + 1, 0);
    p.binrow_ptr.assign(p.n_live + 1, 0);
    for (int m = 0; m < p.n_mels; ++m) {
        for (int k = 0; k < p.F; ++k) {
            const float v = p.fb[static_cast<size_t>(k) * p.n_mels + m];
            if (v != 0.0f) {
                p.melcol_j.push_back(p.jofk[k]);
                p.melcol_w.push_back(v);
            }
        }
        p.melcol_ptr[m + 1] = static_cast<int32_t>(p.melcol_j.size());
    }
    for (int j = 0; j < p.n_live; ++j) {
        const int k = p.bins[j];
        for (int m = 0; m < p.n_mels; ++m) {
            const float v = p.fb[static_cast<size_t>(k) * p.n_mels + m];
            if (v != 0.0f) {
                p.binrow_m.push_back(m);
                p.binrow_w.push_back(v);
            }
        }
        p.binrow_ptr[j + 1] = static_cast<int32_t>(p.binrow_m.size());
    }

    // ---- Gram matrix (must be tridiagonal) + Thomas factors, fp64
    p.tri.assign(static_cast<size_t>(3) * p.n_mels, 0.0);
    bool tridiag = true;
    for (int k = 0; k < p.F && tridiag; ++k) {
        int first = -1, last = -1;
        for (int m = 0; m < p.n_mels; ++m)
            if (p.fb[static_cast<size_t>(k) * p.n_mels + m] != 0.0f) {
                if (first < 0) first = m;
                last = m;
            }
        if (first >= 0 && last - first > 1) tridiag = false;
        if (first < 0) continue;
        for (int m = first; m <= last; ++m) {
            const double v = p.fb[static_cast<size_t>(k) * p.n_mels + m];
            p.tri[p.n_mels + m] += v * v;
            if (m + 1 <= last) {
                const double v2 = p.fb[static_cast<size_t>(k) * p.n_mels + m + 1];
                p.tri[2 * p.n_mels + m] += v * v2;      // super[m]   = G[m][m+1]
                p.tri[m + 1] += v * v2;                 // sub[m+1]   = G[m+1][m]
            }
        }
    }
    if (!tridiag) {
        code = RF_ERR_UNSUPPORTED;
        return "rf_plan_create: mel filterbank rows overlap more than two filters; the "
               "inverse-mel kernel needs a tridiagonal fb^T fb";
    }
    p.thomas.assign(static_cast<size_t>(2) * p.n_mels, 0.0);
    {
        const double* sub = &p.tri[0];
        const double* dg = &p.tri[p.n_mels];
        const double* sup = &p.tri[2 * p.n_mels];
        double cprev = 0.0;
        for (int i = 0; i < p.n_mels; ++i) {
            const double den = dg[i] - (i ? sub[i] * cprev : 0.0);
            if (!(std::fabs(den) > 1e-300) || !(dg[i] > 0.0)) {
                code = RF_ERR_INVALID;
                // torchaudio warns here (functional.py:579-584) and gels then assumes full rank
                return "rf_plan_create: at least one mel filterbank has all zero values "
                       "(n_mels too high for n_fft); inverse mel is singular";
            }
            const double c = sup[i] / den;
            p.thomas[i] = c;
            p.thomas[p.n_mels + i] = 1.0 / den;
            cprev = c;
        }
    }
    code = RF_OK;
    return std::string();
}
