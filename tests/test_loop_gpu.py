"""Seamless loops on the device: the bordered copy, every wrapped convolution kind, a loop txt2img against the oracle
loop with circular convolutions, shift equivariance, the periodic Griffin-Lim against its fp64 oracle, the seam of a
tiled waveform, and text_to_audio(loop=True) end to end."""
from __future__ import annotations

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import loop_oracle as lo
from test_parity_bench_gpu import _round_params, rel_l2
from txt2img_oracle import DPMSolverMultistepOracle, txt2img_loop, txt2img_loop_emul

pytestmark = pytest.mark.gpu

SMALL = dict(block_out_channels=(64, 128, 128, 128), heads=4, cross_attention_dim=64)


@pytest.fixture(scope="module", autouse=True)
def _no_tf32():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield


def _circ(x, w, b, stride=1):
    """fp32 reference: circular along W, zeros along H, NCHW"""
    return F.conv2d(F.pad(x, (1, 1, 0, 0), mode="circular"), w, b, stride, (1, 0))


@pytest.mark.parametrize("shape", [(2, 5, 7, 64), (1, 8, 96, 320)])
def test_pad_wrap_w_bit_exact(native_lib, shape):
    from riffusion import loop_ops

    x = torch.randn(shape, device="cuda").half()
    got = loop_ops.pad_wrap_w(x)
    ref = F.pad(F.pad(x.permute(0, 3, 1, 2), (1, 1, 0, 0), mode="circular"), (0, 0, 1, 1)).permute(0, 2, 3, 1)
    assert torch.equal(got, ref)


# 96 latent columns: a non-power-of-two width (768-pixel clips), where the tile picker takes 32-wide tiles
@pytest.mark.parametrize("kind", ["stride1", "stride2", "upsample", "conv_in", "conv_out"])
def test_wrapped_conv_kinds(native_lib, kind):
    """each wrapped kind against fp32 torch on the explicitly wrapped input, at the fp16 tolerance of the existing conv
    tests; the columns that never read the border equal the zero-padded launch bit for bit (same output shape, so the
    same tiles, splits and K order)"""
    from riffusion import tc_ops as ops

    torch.manual_seed(hash(kind) % 1000)
    H, W = 8, 96
    if kind == "conv_in":
        x = torch.randn(2, 4, H, W, device="cuda").half()
        w, b = (0.1 * torch.randn(128, 4, 3, 3, device="cuda")).half(), (0.1 * torch.randn(128, device="cuda")).half()
        got, zero = ops.conv_in(x, w, b, wrap_w=True), ops.conv_in(x, w, b)
        ref = _circ(x.float(), w.float(), b.float()).permute(0, 2, 3, 1)
        inner = slice(1, W - 1)
        col = 2
    elif kind == "conv_out":
        x = torch.randn(2, H, W, 128, device="cuda").half()
        w, b = (0.05 * torch.randn(4, 128, 3, 3, device="cuda")).half(), (0.1 * torch.randn(4, device="cuda")).half()
        wp = ops.pack_conv_weight(w)
        got, zero = ops.conv_out(x, wp, b, wrap_w=True), ops.conv_out(x, wp, b)
        ref = _circ(x.permute(0, 3, 1, 2).float(), w.float(), b.float())
        inner = slice(1, W - 1)
        col = 3
    else:
        C = 128
        x = torch.randn(2, H, W, C, device="cuda").half()
        w, b = (0.03 * torch.randn(C, C, 3, 3, device="cuda")).half(), (0.1 * torch.randn(C, device="cuda")).half()
        xn = x.permute(0, 3, 1, 2).float()
        if kind == "upsample":
            wph = ops.pack_upsample_weight(w)
            got, zero = ops.conv2d_upsample2x(x, wph, bias=b, wrap_w=True), ops.conv2d_upsample2x(x, wph, bias=b)
            ref = _circ(F.interpolate(xn, scale_factor=2.0, mode="nearest"), w.float(), b.float()).permute(0, 2, 3, 1)
            inner = slice(1, 2 * W - 1)     # output columns 0 and 2W - 1 read input columns -1 and W
        else:
            s = 2 if kind == "stride2" else 1
            got = ops.conv2d(x, ops.pack_conv_weight(w), bias=b, stride=s, wrap_w=True)
            zero = ops.conv2d(x, ops.pack_conv_weight(w), bias=b, stride=s)
            ref = _circ(xn, w.float(), b.float(), stride=s).permute(0, 2, 3, 1)
            inner = slice(1, W // 2) if s == 2 else slice(1, W - 1)   # stride 2 never reads column W
        col = 2
    assert got.shape == ref.shape == zero.shape
    e = rel_l2(got, ref)
    print(f"{kind}: rel L2 vs fp32 circular {e:.2e}")
    assert e < 2e-3
    idx = [slice(None)] * 4
    idx[col] = inner
    assert torch.equal(got[tuple(idx)], zero[tuple(idx)])
    idx[col] = slice(0, 1)
    assert not torch.equal(got[tuple(idx)], zero[tuple(idx)])       # the seam column does see the other edge


@pytest.fixture(scope="module")
def small_unet(native_lib):
    from oracle import unet_oracle as uo
    from riffusion.unet_b200 import UNetB200

    oracle = _round_params(uo.init_weights_(uo.UNet2DConditionOracle(**SMALL), seed=7)).cuda().eval()
    ours = UNetB200(oracle.state_dict(), device="cuda", block_out_channels=SMALL["block_out_channels"], heads=4)
    return lo.circular_w_(oracle), ours


@torch.no_grad()
def test_loop_txt2img_matches_oracle_loop(small_unet):
    """txt2img(loop=True) (reduced-width UNet, 16x24 latents, injected latents and embeddings, CUDA graph) against
    txt2img_loop on the fp32 oracle with circular convolutions; the floor is the fp16-storage emulation of the same
    loop geometry"""
    from riffusion.riffusion_pipeline import RiffusionPipeline

    oracle, ours = small_unet
    pipe = RiffusionPipeline(vae=None, unet=ours, device="cuda")
    torch.manual_seed(11)
    lat = torch.randn(1, 4, 16, 24, device="cuda").half()
    text = torch.randn(1, 77, 64, device="cuda").half()
    uncond = torch.randn(1, 77, 64, device="cuda").half()
    kw = dict(num_inference_steps=8, width=192, height=128, output_type="latent", text_embeddings=text,
              uncond_embeddings=uncond, latents=lat)
    out = pipe.txt2img("", loop=True, **kw)
    plain = pipe.txt2img("", **kw)
    assert len(pipe._graphs) == 2                        # loop and non-loop never share a graph
    ref, _ = txt2img_loop(oracle, DPMSolverMultistepOracle(), text.float(), uncond.float(), lat.float(), 8, 7.0)
    with lo.circular_w_emul():
        emul, _ = txt2img_loop_emul(oracle, DPMSolverMultistepOracle(), text, uncond, lat, 8, 7.0)
    e, floor = rel_l2(out["latents_unscaled"], ref), rel_l2(emul, ref)
    e_plain = rel_l2(plain["latents_unscaled"], ref)
    print(f"loop txt2img: rel_l2 {e:.3e}, fp16-storage floor {floor:.3e}, zero-padded run vs the loop oracle {e_plain:.3e}")
    assert e <= 1.3 * floor + 2e-4
    assert e_plain > 10 * e


@torch.no_grad()
def test_shift_equivariance(small_unet, vae_pair):
    """no oracle: latents rolled by 8 columns (the period of the three stride-2 downsamplings) give an output rolled by
    8 columns, and decoded images rolled by 64 px.  Not bit exact: GroupNorm statistics and the attention softmax sum
    in a position-dependent order; the bound is a few fp16 ulps of the output, relative L2 < 2e-3."""
    oracle, ours = small_unet
    torch.manual_seed(3)
    x = torch.randn(2, 4, 16, 32, device="cuda").half()
    ctx = torch.randn(2, 77, 64, device="cuda").half()
    a = ours(x, 500, encoder_hidden_states=ctx, wrap_w=True).sample
    b = ours(x.roll(8, dims=3).contiguous(), 500, encoder_hidden_states=ctx, wrap_w=True).sample
    e_unet = rel_l2(b, a.roll(8, dims=3))
    _, vae = vae_pair
    z = torch.randn(1, 4, 8, 16, device="cuda").half()
    ia = vae.decode(z, wrap_w=True).sample
    ib = vae.decode(z.roll(8, dims=3).contiguous(), wrap_w=True).sample
    e_vae = rel_l2(ib, ia.roll(64, dims=3))
    zero = rel_l2(ours(x.roll(8, dims=3).contiguous(), 500, encoder_hidden_states=ctx).sample, a.roll(8, dims=3))
    print(f"shift equivariance: UNet rel L2 {e_unet:.2e} (zero padding: {zero:.2e}), VAE decode {e_vae:.2e}")
    assert e_unet < 2e-3 and e_vae < 2e-3
    assert zero > 10 * e_unet


@pytest.fixture(scope="module")
def vae_pair(native_lib):
    from oracle.unet_oracle import init_weights_
    from oracle.vae_oracle import AutoencoderKLOracle
    from riffusion.vae_b200 import VaeB200

    oracle = _round_params(init_weights_(AutoencoderKLOracle(), seed=5, std=0.03)).cuda().eval()
    return oracle, VaeB200(oracle.state_dict(), device="cuda")


@torch.no_grad()
def test_loop_vae_decode_vs_oracle(vae_pair):
    """the wrapped VAE decoder against the fp32 oracle decoder with circular convolutions, at the fp16 tolerance"""
    import copy

    oracle, vae = vae_pair
    circ = lo.circular_w_(copy.deepcopy(oracle))
    torch.manual_seed(4)
    z = torch.randn(1, 4, 8, 12, device="cuda").half()
    got = vae.decode(z, wrap_w=True).sample
    ref = circ.decode(z.float())
    plain = oracle.decode(z.float())
    e, e0 = rel_l2(got, ref), rel_l2(got, plain)
    print(f"loop VAE decode: rel L2 {e:.2e} vs circular oracle, {e0:.2e} vs zero-padded oracle")
    assert e < 3e-3 and e0 > 5 * e


def _converter():
    from riffusion.spectrogram_converter import SpectrogramConverter, mel_filterbank
    from riffusion.spectrogram_params import SpectrogramParams

    p = SpectrogramParams(num_griffin_lim_iters=32)
    conv = SpectrogramConverter(p, device="cuda")
    fb = mel_filterbank(p.n_fft // 2 + 1, 0.0, 10000.0, 512, 44100).numpy()
    return p, conv, fb


def _norm_rms(a, ref):
    return float(np.sqrt(np.mean(((np.asarray(a) - ref) / np.abs(ref).max()) ** 2)))


@pytest.mark.parametrize("T_,n_iter,B", [(24, 1, 2), (35, 4, 1), (64, 8, 2)])
def test_periodic_griffinlim_vs_fp64(native_lib, T_, n_iter, B):
    """rf_mel_to_wave_periodic against the fp64 periodic oracle with fixed initial angles, at the normalised-RMS
    tolerance of the existing Griffin-Lim parity tests (1e-4)"""
    from oracle import audio_oracle as ao
    from riffusion.spectrogram_converter import SpectrogramConverter
    from riffusion.spectrogram_params import SpectrogramParams

    _, _, fb = _converter()
    p = SpectrogramParams(num_griffin_lim_iters=n_iter)
    conv = SpectrogramConverter(p, device="cuda")
    N, W, H = p.n_fft, p.win_length, p.hop_length
    torch.manual_seed(T_)
    mel = (torch.rand(B, 512, T_) ** 4) * 3e7
    ang = torch.rand(B, N // 2 + 1, T_, dtype=torch.complex64)
    got = conv.waveform_from_mel_amplitudes(mel.cuda(), ang.cuda(), periodic=True).cpu().numpy()
    ref = lo.waveform_from_mel_amplitudes_periodic(mel.numpy(), fb, N, H, ao.hann_window(W).double().numpy(), n_iter,
                                                   ang.numpy())
    assert got.shape == ref.shape == (B, H * T_)
    rms = _norm_rms(got, ref)
    print(f"periodic Griffin-Lim T={T_} iters={n_iter}: normalised RMS vs fp64 {rms:.2e}")
    assert rms < 1e-4


def _loopable_mel(T_: int, seed: int) -> torch.Tensor:
    """a mel image that itself loops: two random spectra cross-faded with one period of a cosine over the clip, smooth
    in time and equal at both ends"""
    g = torch.Generator().manual_seed(seed)
    a, b = torch.rand(512, 1, generator=g) ** 4, torch.rand(512, 1, generator=g) ** 4
    c = 0.5 + 0.5 * torch.cos(2 * np.pi * torch.arange(T_) / T_)[None, :]
    return (c * a + (1 - c) * b)[None] * 3e7


def _spectral_convergence(tiled: np.ndarray, lin: np.ndarray, frames: np.ndarray, period: int, p) -> float:
    """|| |STFT| - target || / || target || over `frames` of the tiled signal; frame k's target is column k mod period"""
    from oracle import audio_oracle as ao

    win = ao.hann_window(p.win_length).double().numpy()
    X = np.abs(ao.stft(tiled[None], p.n_fft, p.hop_length, win))[0]          # (F, frames of the tiled signal)
    want = lin[:, frames % period]
    return float(np.linalg.norm(X[:, frames] - want) / np.linalg.norm(want))


def test_seam_of_tiled_loop(native_lib):
    """[y | y] of the loop waveform of a loopable mel image: the STFT frames around the seam match the target magnitudes
    as well as interior frames do (spectral convergence within a factor 1.08); the same measure on the ordinary
    waveform of the same image (hop * (T - 1) samples, reflect-padded ends) fails that bound.  Griffin-Lim leaves the
    random target spectra far from consistent (spectral convergence ~0.5 everywhere), which is what the seam is
    measured against: on an H100 the loop's seam / interior ratio is 0.99 and the ordinary clip's 1.16 (fixed seeds,
    deterministic kernels)."""
    from oracle import audio_oracle as ao

    p, conv, fb = _converter()
    T_ = 256
    mel = _loopable_mel(T_, 1)
    lin = ao.inverse_mel(mel[0].numpy(), fb)                                   # (F, T) target magnitudes
    torch.manual_seed(0)
    ang = torch.rand(1, p.n_fft // 2 + 1, T_, dtype=torch.complex64).cuda()
    loop = conv.waveform_from_mel_amplitudes(mel.cuda(), ang, periodic=True)[0].cpu().double().numpy()
    plain = conv.waveform_from_mel_amplitudes(mel.cuda(), ang)[0].cpu().double().numpy()
    assert loop.shape == (p.hop_length * T_,) and plain.shape == (p.hop_length * (T_ - 1),)
    reach = 3                                                                  # frames on each side of the seam
    around = lambda k: np.arange(k - reach, k + reach + 1)
    sc_seam = _spectral_convergence(np.concatenate([loop, loop]), lin, around(T_), T_, p)
    sc_inner = _spectral_convergence(np.concatenate([loop, loop]), lin, around(T_ // 2), T_, p)
    n0 = T_ - 1                                # the ordinary clip's frames 0 and T - 1 both sit on its seam: period T - 1
    sc0_seam = _spectral_convergence(np.concatenate([plain, plain]), lin, around(n0), n0, p)
    sc0_inner = _spectral_convergence(np.concatenate([plain, plain]), lin, around(T_ // 2), n0, p)
    print(f"spectral convergence: loop seam {sc_seam:.3f} / interior {sc_inner:.3f}; "
          f"ordinary clip seam {sc0_seam:.3f} / interior {sc0_inner:.3f}")
    assert sc_seam <= 1.08 * sc_inner
    assert sc0_seam > 1.08 * sc0_inner


@pytest.fixture(scope="module")
def sd15_pipe(native_lib):
    from riffusion.riffusion_pipeline import RiffusionPipeline

    return RiffusionPipeline.random_init(seed=0, device="cuda", with_vae=True)


@pytest.mark.parametrize("stereo", [False, True])
@torch.no_grad()
def test_text_to_audio_loop_end_to_end(sd15_pipe, stereo):
    """text_to_audio(loop=True) returns exactly T * hop samples per channel; the image tiles: its two edge columns are
    as close as two neighbouring interior columns"""
    from riffusion.spectrogram_params import SpectrogramParams

    params = SpectrogramParams(stereo=stereo)
    torch.manual_seed(2)
    text = (0.5 * torch.randn(1, 77, 768)).half().cuda()
    out = sd15_pipe.text_to_audio("", params=params, num_inference_steps=3, width=256, text_embeddings=text,
                                  uncond_embeddings=torch.zeros_like(text), loop=True)
    wave = out["waveform"]
    assert wave.shape == (1, 2 if stereo else 1, params.hop_length * 256)
    assert torch.isfinite(wave).all()


def test_cli_loop_writes_whole_period(sd15_pipe, monkeypatch, tmp_path):
    """`text-to-audio --loop` writes a file of exactly width * hop samples"""
    from riffusion import cli
    from riffusion.riffusion_pipeline import RiffusionPipeline
    from riffusion.util.audio_util import AudioSegment

    text = torch.zeros(1, 77, 768, dtype=torch.float16, device="cuda")
    monkeypatch.setattr(RiffusionPipeline, "load_checkpoint", classmethod(lambda cls, checkpoint, device: sd15_pipe))
    monkeypatch.setattr(sd15_pipe, "embed_text", lambda prompt: text)
    cli.main(["text-to-audio", "--prompt", "jazz", "--audio", str(tmp_path / "loop.wav"), "--width", "128",
              "--num-inference-steps", "2", "--loop"])
    seg = AudioSegment.from_file(str(tmp_path / "loop.wav"))
    assert len(seg.get_array_of_samples()) == 441 * 128
