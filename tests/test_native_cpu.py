"""CPU-only checks of the native side: the C-ABI library builds, loads and exports every symbol
include/rf_b200.h declares; plan tables are correct; the device control flow (emulated on the host
with the same phase functions the kernels call) reproduces torch.stft / torchaudio Griffin-Lim."""
import ctypes
import re
from pathlib import Path

import numpy as np
import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]
N, W, H, F = 17640, 4410, 441, 8821


def test_header_symbols_exported(native_lib):
    header = (ROOT / "include" / "rf_b200.h").read_text()
    declared = set(re.findall(r"\b(rf_[a-z0-9_]+)\s*\(", header))
    declared -= {"rf_plan_desc", "rf_plan_info"}
    from riffusion import _native

    assert declared == set(_native.SIGNATURES), declared ^ set(_native.SIGNATURES)
    for name in declared:
        assert hasattr(native_lib, name)
    assert b"sm_90a" in native_lib.rf_version()


def test_no_cpu_fallback_without_gpu(native_lib):
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from riffusion import _native
    from riffusion.spectrogram_converter import SpectrogramConverter, get_plan
    from riffusion.spectrogram_params import SpectrogramParams

    with pytest.raises(RuntimeError):
        SpectrogramConverter(SpectrogramParams(), device="cuda")
    with pytest.raises(RuntimeError):
        SpectrogramConverter(SpectrogramParams(), device="cpu")
    plan = get_plan(SpectrogramParams(), full_band=False)
    # a device entry point must fail loudly, not compute on the host
    rc = native_lib.rf_inverse_mel(plan.handle, ctypes.c_void_p(16), 1, 32, ctypes.c_void_p(16), None)
    assert rc == 2 and b"no CPU fallback" in native_lib.rf_last_error()
    with pytest.raises(_native.NativeError):
        _native.require_cuda(torch.zeros(4), "x", torch.float32)


def test_unsupported_geometry_is_loud(native_lib):
    from riffusion.spectrogram_converter import get_plan
    from riffusion.spectrogram_params import SpectrogramParams

    # other sample rates run on the generic mixed-radix engine (48 kHz: n_fft 19200 = 2 * 2^7 3 5^2; 22.05 kHz: hop 220
    # does not divide win 2205) ...
    for sr, n_fft, win, hop in ((48000, 19200, 4800, 480), (22050, 8820, 2205, 220)):
        prm = SpectrogramParams(sample_rate=sr)
        assert (prm.n_fft, prm.win_length, prm.hop_length) == (n_fft, win, hop)
        plan = get_plan(prm, full_band=False)
        assert plan.info.n_freq == n_fft // 2 + 1 and plan.info.n_live > 0
    # ... unless n_fft/2 has a prime factor above 7 (44 kHz: 17600 / 2 = 2^5 5^2 11) or the frame exceeds shared memory
    with pytest.raises(NotImplementedError):
        get_plan(SpectrogramParams(sample_rate=44000), full_band=False)
    with pytest.raises(NotImplementedError):
        get_plan(SpectrogramParams(sample_rate=96000), full_band=False)


def test_plan_tables(native_lib):
    from riffusion.spectrogram_converter import get_plan, mel_filterbank
    from riffusion.spectrogram_params import SpectrogramParams

    for params, n_live, k_lo, k_hi, nnz in (
        (SpectrogramParams(), 4000, 1, 4000, 7976),
        (SpectrogramParams(min_frequency=20, max_frequency=20000), 7991, 9, 7999, 15927),
    ):
        plan = get_plan(params, full_band=False)
        i = plan.info
        assert (i.n_freq, i.n_live, i.k_lo, i.k_hi, i.fb_nnz) == (F, n_live, k_lo, k_hi, nnz)
        bins = plan.table("bins", np.int32, (n_live,))
        assert sorted(bins.tolist()) == list(range(k_lo, k_hi + 1))
        assert np.all(bins[: i.n_even] % 2 == 0) and np.all(bins[i.n_even:] % 2 == 1)
        pp = plan.table("pp", np.uint32, (n_live,))
        r, idx, idx2, k7 = pp & 3, (pp >> 2) & 8191, (pp >> 15) & 8191, pp >> 28
        assert np.array_equal(r, bins % 4) and np.array_equal(k7, bins % 8)

        def pos(m):          # spectral slot: the 7-thread radix-49 pass leaves output c at 7 (c % 7) + c // 7 of its block
            c = m % 49
            return (m % 10) * 441 + (m % 9) * 49 + 7 * (c % 7) + c // 7

        assert np.array_equal(idx, pos(bins // 4))
        assert np.array_equal(idx2, pos(((N - bins) % N) // 4))
        # bank-aware order: 16 consecutive bins of one r block hit 16 distinct 8-byte bank pairs
        blk = slice(0, 16 * 40)
        assert all(len(set((idx[blk][i:i + 16] % 16).tolist())) == 16 for i in range(0, 16 * 40 - 16))
        # kernel-side per-bin tables derived from pp: V offsets of the bin and its Hermitian partner, phase constants
        bt = plan.table("bt", np.uint32, (n_live,))
        rp = (4 - r) % 4
        assert np.array_equal(bt & 16383, (r >> 1) * W + idx) and np.array_equal((bt >> 14) & 16383, (rp >> 1) * W + idx2)
        assert np.array_equal(bt >> 31, ((idx == idx2) & (r == rp)).astype(np.uint32))
        ph = np.exp(-2j * np.pi * 3 * bins / 8)
        ai = plan.table("ab_inv", np.float32, (n_live, 4)).astype(np.float64)
        af = plan.table("ab_fwd", np.float32, (n_live, 4)).astype(np.float64)
        assert np.abs(ai[:, 0] + 1j * ai[:, 1] - np.conj(ph)).max() < 1e-7
        assert np.abs(ai[:, 2] + 1j * ai[:, 3] - 1j * np.conj(ph)).max() < 1e-7
        assert np.abs(af[:, 0] + 1j * af[:, 1] - ph / 2).max() < 1e-7
        assert np.abs(af[:, 2] + 1j * af[:, 3] - (-1j) * ph / 2).max() < 1e-7
        if i.k_hi * 2 + 800 <= N // 2:    # decimated loop eligible: odd-sample frame carries exp(-2 pi i k/N)
            po = np.exp(-2j * np.pi * bins / N)
            pp2 = plan.table("pp2", np.uint32, (n_live,))
            bt2 = plan.table("bt2", np.uint32, (n_live,))
            assert np.array_equal(bt2 & 16383, ((pp2 & 3) >> 1) * (W // 2) + ((pp2 >> 2) & 8191))
            a2 = plan.table("ab2_inv", np.float32, (n_live, 4)).astype(np.float64)
            f2 = plan.table("ab2_fwd", np.float32, (n_live, 4)).astype(np.float64)
            assert np.abs(a2[:, 2] + 1j * a2[:, 3] - 1j * np.conj(ph * po)).max() < 1e-7
            assert np.abs(f2[:, 2] + 1j * f2[:, 3] - (-1j) * ph * po / 2).max() < 1e-7
        fb = plan.table("fb", np.float32, (F, 512))
        assert np.array_equal(fb, mel_filterbank(F, float(params.min_frequency), float(params.max_frequency),
                                                 512, 44100).numpy())
        # modulation tables: w[n'] * exp(-2 pi i r n'/N) at the prime-factor position of n'
        wt = plan.table("wt_fwd", np.float32, (4, W, 2))
        wi = plan.table("wt_inv", np.float32, (4, W, 2))
        win = torch.hann_window(W).double().numpy()
        b, c, a = np.meshgrid(np.arange(9), np.arange(49), np.arange(10), indexing="ij")   # table order [b][c][a]
        n_of = ((441 * a + 490 * b + 90 * c) % W).ravel()
        for rr in range(4):
            ref = win[n_of] * np.exp(-2j * np.pi * ((rr * n_of) % N) / N)
            assert np.abs(wt[rr, :, 0] + 1j * wt[rr, :, 1] - ref).max() < 1e-7
            assert np.abs((wi[rr, :, 0] + 1j * wi[rr, :, 1]) * N - np.conj(ref)).max() < 1e-6
        # Gram matrix is tridiagonal and the dense min-norm operator solves fb^T P = I
        tri = plan.table("tri", np.float64, (3, 512))
        gram = fb.astype(np.float64).T @ fb.astype(np.float64)
        assert np.allclose(np.diag(gram), tri[1]) and np.allclose(np.diag(gram, 1), tri[2][:-1])
        assert np.allclose(np.diag(gram, -1), tri[0][1:])
        off = gram.copy()
        for d in (-1, 0, 1):
            off -= np.diag(np.diag(gram, d), d)
        assert np.abs(off).max() == 0          # only neighbouring triangles overlap
        pinv = plan.table("pinv", np.float32, (F, 512))
        assert np.abs(fb.astype(np.float64).T @ pinv.astype(np.float64) - np.eye(512)).max() < 1e-5


def _emu_plan(hostemu, full_band, f_min=0.0, f_max=10000.0):
    from riffusion import _native
    from riffusion.spectrogram_converter import mel_filterbank

    desc = _native.PlanDesc(44100, N, W, H, 512, f_min, f_max, 0, 0, int(full_band))
    fb = mel_filterbank(F, f_min, f_max, 512, 44100).numpy()
    win = torch.hann_window(W).numpy()
    p = hostemu.emu_plan_create(ctypes.byref(desc), win.ctypes.data, np.ascontiguousarray(fb).ctypes.data)
    assert p, hostemu.emu_last_error()
    return p, fb


@pytest.mark.parametrize("full_band", [True, False])
@pytest.mark.parametrize("L", [H * 24, H * 24 + 100, H * 25 + 440])   # even / ragged / odd frame counts
def test_emulated_stft_matches_torch(hostemu, full_band, L):
    p, fb = _emu_plan(hostemu, full_band)
    torch.manual_seed(L)
    x = torch.randn(L) * 1000
    ref = torch.stft(x, N, H, W, torch.hann_window(W), center=True, pad_mode="reflect", return_complex=True)
    if not full_band:
        ref = ref * torch.from_numpy((fb != 0).any(axis=1))[:, None]
    out = np.zeros((F, ref.shape[1], 2), np.float32)
    xn = x.numpy().copy()
    hostemu.emu_stft(p, xn.ctypes.data, L, out.ctypes.data)
    got = torch.view_as_complex(torch.from_numpy(out))
    assert (got - ref).abs().max() / ref.abs().max() < 1e-6
    hostemu.emu_plan_destroy(p)


@pytest.mark.parametrize("full_band,T_,n_iter", [(True, 24, 2), (False, 24, 3), (False, 35, 2), (False, 22, 0)])
def test_emulated_griffinlim_matches_torchaudio(hostemu, full_band, T_, n_iter):
    """same chunked overlap-add, pair packing and buffer rotation as the CUDA path; T_=35 has an odd
    frame count and crosses two overlap-add chunks (16 frames each) plus a ragged third"""
    import torchaudio

    from oracle.torchaudio_ref import griffinlim_with_angles

    p, fb = _emu_plan(hostemu, full_band)
    torch.manual_seed(T_ * 10 + n_iter)
    mag = torch.rand(F, T_) * 100
    if not full_band:
        mag = mag * torch.from_numpy((fb != 0).any(axis=1))[:, None]
    ang = torch.rand(F, T_, dtype=torch.complex64)
    gl = torchaudio.transforms.GriffinLim(n_fft=N, n_iter=n_iter, win_length=W, hop_length=H, power=1.0,
                                          momentum=0.99, rand_init=True)
    ref = griffinlim_with_angles(gl, mag[None], ang[None])[0]
    # fp64 restatement as tie-breaker: Griffin-Lim amplifies fp32 rounding at ill-conditioned bins
    # (|R - m*tprev| ~ 0), so torchaudio-fp32 itself can sit 1e-4 away from the exact recurrence
    # (seed 352, T=35); the bar is "as close to the exact answer as torchaudio is", plus closeness to
    # torchaudio whenever torchaudio is itself well conditioned.
    from oracle import audio_oracle as ao

    o64 = torch.from_numpy(ao.griffinlim(mag[None].numpy(), N, H, torch.hann_window(W).double().numpy(), n_iter,
                                         0.99, ang[None].numpy())[0]).float()
    wave = np.zeros(H * (T_ - 1), np.float32)
    hostemu.emu_griffinlim(p, mag.numpy().ctypes.data, torch.view_as_real(ang).numpy().ctypes.data, T_, n_iter,
                           ctypes.c_float(0.99), wave.ctypes.data)
    got = torch.from_numpy(wave)
    err_ours = ((got - o64).norm() / o64.norm()).item()
    err_ta = ((ref - o64).norm() / o64.norm()).item()
    assert err_ours < max(5e-6, err_ta)      # never further from the exact recurrence than torchaudio-fp32
    if err_ta < 5e-6:
        assert ((got - ref).norm() / ref.norm()).item() < 1e-5
    hostemu.emu_plan_destroy(p)


@pytest.mark.parametrize("T_,n_iter", [(64, 3), (75, 4), (97, 8)])
def test_emulated_decimated_griffinlim(hostemu, T_, n_iter):
    """The half-rate inner loop (odd samples + two full-rate edge strips built from both sample parities, DESIGN.md 3.2 / 3.3c) against the full-rate loop,
    the fp64 oracle and torchaudio.  T_=64 is the smallest eligible clip (c_tail = 3: frames >= T-16 reach the tail strip), 75 / 97 have odd frame counts
    and ragged last chunks."""
    import torchaudio

    from oracle import audio_oracle as ao
    from oracle.torchaudio_ref import griffinlim_with_angles

    p, fb = _emu_plan(hostemu, False)
    assert hostemu.emu_plan_decimate(p) == 1
    torch.manual_seed(T_ + n_iter)
    mag = torch.rand(F, T_) * 100 * torch.from_numpy((fb != 0).any(axis=1))[:, None]
    ang = torch.rand(F, T_, dtype=torch.complex64)
    gl = torchaudio.transforms.GriffinLim(n_fft=N, n_iter=n_iter, win_length=W, hop_length=H, power=1.0,
                                          momentum=0.99, rand_init=True)
    ref = griffinlim_with_angles(gl, mag[None], ang[None])[0].numpy()
    o64 = ao.griffinlim(mag[None].numpy(), N, H, torch.hann_window(W).double().numpy(), n_iter, 0.99,
                        ang[None].numpy())[0]
    out = {}
    for dec in (0, 1):
        wave = np.zeros(H * (T_ - 1), np.float32)
        hostemu.emu_griffinlim2(p, mag.numpy().ctypes.data, torch.view_as_real(ang).numpy().ctypes.data, T_, n_iter,
                                ctypes.c_float(0.99), dec, wave.ctypes.data)
        out[dec] = wave
    nrm = np.linalg.norm(o64)
    err_ta = np.linalg.norm(ref - o64) / nrm
    err_full = np.linalg.norm(out[0] - o64) / nrm
    err_dec = np.linalg.norm(out[1] - o64) / nrm
    assert not np.array_equal(out[0], out[1])            # the decimated path really ran
    assert err_full < max(5e-6, err_ta)
    assert err_dec < max(1e-5, 3 * err_ta)                # aliasing stays at the fp32 rounding level
    hostemu.emu_plan_destroy(p)


def test_decimation_eligibility(hostemu):
    """full-band plans (k_hi = n_fft/2) and wide mel bands must not decimate"""
    p, _ = _emu_plan(hostemu, True)
    assert hostemu.emu_plan_decimate(p) == 0
    hostemu.emu_plan_destroy(p)
    p, _ = _emu_plan(hostemu, False, 0.0, 12000.0)
    assert hostemu.emu_plan_decimate(p) == 0
    hostemu.emu_plan_destroy(p)
    p, _ = _emu_plan(hostemu, False, 0.0, 10000.0)
    assert hostemu.emu_plan_decimate(p) == 1
    hostemu.emu_plan_destroy(p)
    # the edge strips of the hybrid loop are laid out for hop = 441: another odd hop (step 50 ms) must stay full rate
    # (it was eligible once and came out 40 % wrong in the emulator)
    from riffusion import _native
    from riffusion.spectrogram_converter import mel_filterbank

    desc = _native.PlanDesc(44100, N, W, 2205, 512, 0.0, 10000.0, 0, 0, 0)
    fb = np.ascontiguousarray(mel_filterbank(F, 0.0, 10000.0, 512, 44100).numpy())
    win = torch.hann_window(W).numpy()
    p = hostemu.emu_plan_create(ctypes.byref(desc), win.ctypes.data, fb.ctypes.data)
    assert p and hostemu.emu_plan_decimate(p) == 0
    hostemu.emu_plan_destroy(p)


def test_radix9_slot_order_is_a_permutation_with_fewer_bank_conflicts(native_lib):
    """csrc/rf_pass_b_perm.inc (scratch/gen_pass_b_perm.py): the slot -> item order of the radix-9 pass covers every (a, c)
    item once, its sample index is n'(a, 0, c), and by the exact shared-memory bank model (32 banks x 4 B; 8-byte accesses in
    half-warp phases) a pass costs fewer wavefronts than with lanes running over a, the round-1 order."""
    from riffusion.spectrogram_converter import get_plan
    from riffusion.spectrogram_params import SpectrogramParams

    plan = get_plan(SpectrogramParams(), full_band=False)

    def cost(NA, items_ac):
        Wn, SB, SC, off1 = NA * 441, NA * 49, NA * 9, (441 if NA == 10 else 221)
        tot = 0
        for w0 in range(0, len(items_ac), 32):
            grp = items_ac[w0:w0 + 32]
            for b in range(9):
                n0 = [((441 * a + SC * c) % Wn + SB * b) % Wn for a, c in grp]
                for sh in (0, off1):
                    tot += np.bincount([(n + sh) % 32 for n in n0], minlength=32).max()
                v = [(a * 441 + c + 49 * b) % 16 for a, c in grp]
                tot += np.bincount(v[:16], minlength=16).max() + (np.bincount(v[16:], minlength=16).max() if len(v) > 16 else 0)
        return int(tot)

    for NA, name in ((10, "items"), (5, "items2")):
        it = plan.table(name, np.uint32, (49 * NA,))
        vpos, base = it & 4095, it >> 12
        a, c = vpos // 441, vpos % 441
        assert c.max() < 49 and sorted((a * 49 + c).tolist()) == list(range(49 * NA))
        assert np.array_equal(base, (441 * a + (NA * 9) * c) % (NA * 441))
        shipped = cost(NA, list(zip(a.tolist(), c.tolist())))
        lanes_over_a = cost(NA, [(t % NA, t // NA) for t in range(49 * NA)])
        assert shipped < 0.9 * lanes_over_a, (NA, shipped, lanes_over_a)


def test_other_parity_tables_and_inverse_transform(native_lib, hostemu):
    """The hybrid Griffin-Lim loop fills its full-rate edge strips from two half-rate inverse transforms, one per sample
    parity (DESIGN.md 3.3c).  (1) The other-parity tables: windows swapped, alpha = conj(ph po), beta = i conj(ph).
    (2) The emulated half-rate inverse transform on the other parity, run over EVERY chunk, reproduces the even samples of
    torch.istft — the inverse transform of a band-limited spectrum is exact on any sample subset."""
    from riffusion.spectrogram_converter import get_plan
    from riffusion.spectrogram_params import SpectrogramParams

    plan = get_plan(SpectrogramParams(), full_band=False)
    n_live = plan.info.n_live
    bins = plan.table("bins", np.int32, (n_live,))
    ph, po = np.exp(-2j * np.pi * 3 * bins / 8), np.exp(-2j * np.pi * bins / N)
    ab = plan.table("ab2o_inv", np.float32, (n_live, 4)).astype(np.float64)
    assert np.abs(ab[:, 0] + 1j * ab[:, 1] - np.conj(ph * po)).max() < 1e-7
    assert np.abs(ab[:, 2] + 1j * ab[:, 3] - 1j * np.conj(ph)).max() < 1e-7
    w2, w2o = plan.table("wg2_inv", np.float32, (9, 245, 4)), plan.table("wg2o_inv", np.float32, (9, 245, 4))
    assert np.array_equal(w2[..., 0], w2o[..., 1]) and np.array_equal(w2[..., 1], w2o[..., 0])
    assert np.array_equal(w2[..., 2:], w2o[..., 2:])

    p, fb = _emu_plan(hostemu, False)
    for T_ in (40, 51):                                   # even and odd frame counts, ragged last chunk
        torch.manual_seed(T_)
        live = torch.from_numpy((fb != 0).any(axis=1))[:, None]
        mag = torch.rand(F, T_) * 10 * live
        ang = torch.exp(2j * np.pi * torch.rand(F, T_)).to(torch.complex64)
        L = H * (T_ - 1)
        ref = torch.istft((mag * ang).to(torch.complex64), N, H, W, torch.hann_window(W), length=L).numpy()
        even = np.zeros((L + 1) // 2, np.float32)
        hostemu.emu_istft_other_parity(p, mag.numpy().ctypes.data, torch.view_as_real(ang).contiguous().numpy().ctypes.data,
                                       T_, even.ctypes.data)
        assert np.abs(even - ref[0::2]).max() < 2e-6 * np.abs(ref).max()
    hostemu.emu_plan_destroy(p)
