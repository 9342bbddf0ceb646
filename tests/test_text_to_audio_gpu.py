"""Text-to-audio on the H100: the fused guidance + DPM-Solver++ kernel against fp64, the convolution tiles of
non-power-of-two widths, the SD-1.5-width UNet and VAE at 64x96 latents, txt2img loops against the oracle loop, graph
replay / batching / seeds, text_to_audio end to end judged stage by stage, and the `text-to-audio` command.

Bars are those of tests/test_parity_bench_gpu.py: whole-network outputs within 1.15 x the fp16-storage floor (+1e-4)
of the fp32 oracle, loops within 1.3 x the floor of the loop (+2e-4)."""
import numpy as np
import pytest
import torch

from test_parity_bench_gpu import _check_vs_floor, _round_params, rel_l2
from txt2img_oracle import DPMSolverMultistepOracle, txt2img_loop, txt2img_loop_emul

pytestmark = pytest.mark.gpu

SMALL = dict(block_out_channels=(64, 128, 128, 128), heads=4, cross_attention_dim=64)


@pytest.fixture(scope="module", autouse=True)
def _no_tf32():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield


@pytest.fixture(scope="module")
def small_unet(native_lib):
    from oracle import unet_oracle as uo
    from riffusion.unet_b200 import UNetB200

    oracle = _round_params(uo.init_weights_(uo.UNet2DConditionOracle(**SMALL), seed=7)).cuda().eval()
    return oracle, UNetB200(oracle.state_dict(), device="cuda", block_out_channels=SMALL["block_out_channels"], heads=4)


@pytest.fixture(scope="module")
def vae_pair(native_lib):
    from oracle.unet_oracle import init_weights_
    from oracle.vae_oracle import AutoencoderKLOracle
    from riffusion.vae_b200 import VaeB200

    oracle = _round_params(init_weights_(AutoencoderKLOracle(), seed=5, std=0.03)).cuda().eval()
    return oracle, VaeB200(oracle.state_dict(), device="cuda")


# ----------------------------------------------------------------------------------------------- G1
@pytest.mark.parametrize("second_order", [False, True])
def test_cfg_dpmpp_step_kernel(native_lib, second_order):
    """guided eps bit-identical to torch's fp16 expression; x0 and x' within one fp16 rounding + 2^-20 relative of an
    fp64 evaluation (x' from the kernel's own fp16 x0, the value it stores and the next step reads back); shape
    (2,4,64,65) so that the element count is not a multiple of 8"""
    from riffusion import tc_ops as ops
    from riffusion.scheduler_b200 import DPMSolverMultistepSchedulerB200

    torch.manual_seed(31 + second_order)
    shape = (2, 4, 64, 65)
    pair = torch.randn((4,) + shape[1:], device="cuda").half()
    x = (torch.randn(shape, device="cuda") * 3).half()
    m1 = torch.randn(shape, device="cuda").half() if second_order else None
    sched = DPMSolverMultistepSchedulerB200()
    sched.set_timesteps(30)
    sched.lower_order_nums = 1 if second_order else 0
    order, coefs = sched.plan(int(sched.timesteps[5]))
    assert order == (2 if second_order else 1)
    g = 7.5
    x0, prev = ops.cfg_dpmpp_step(pair, g, x, m1, coefs)
    eu, et = pair[:2], pair[2:]
    eps = eu + g * (et - eu)                                            # torch fp16 arithmetic
    a, s, c_x, c_0, c_1 = (float(np.float32(v)) for v in coefs)         # the fp32 values the kernel receives
    x0_64 = (x.double() - s * eps.double()) / a
    ulp = lambda v: torch.finfo(torch.float16).eps * v.abs().clamp_min(2.0 ** -14)       # noqa: E731
    err0 = (x0.double() - x0_64).abs()
    assert bool((err0 <= 0.5 * ulp(x0_64) + 2.0 ** -20 * (x.double().abs() + abs(s) * eps.double().abs()) / a).all())
    x0h = x0.double()
    p64 = c_x * x.double() + c_0 * x0h
    mag = (c_x * x.double()).abs() + (c_0 * x0h).abs()
    if second_order:
        p64 = p64 + c_1 * (x0h - m1.double())
        mag = mag + (c_1 * (x0h - m1.double())).abs()
    err = (prev.double() - p64).abs()
    assert bool((err <= 0.5 * ulp(p64) + 2.0 ** -20 * mag).all())
    # the guided eps is the fp16 torch expression bit for bit: a step with sigma = 0, alpha = 1 passes x through, and
    # with x = 0, sigma = -1, alpha = 1 x0 equals the guided eps exactly
    x0e, _ = ops.cfg_dpmpp_step(pair, g, torch.zeros_like(x), None, (1.0, -1.0, 1.0, 0.0, 0.0))
    assert torch.equal(x0e, eps)


# ----------------------------------------------------------------------------------------------- G2
@pytest.mark.parametrize("W", [96, 48, 24, 12, 20])
def test_conv_tiles_non_power_of_two_widths(native_lib, W):
    """rf_conv2d_f16 at H = 64 and widths whose tile width changes (96 -> 32, 48 -> 16, 24 -> 8, 20 -> 8) or not (12):
    3x3 stride 1 and 2, 1x1, two-input concatenation and the fused nearest-2x upsample, against torch fp32 on the
    same fp16 inputs at the bar of tests/test_tc_gpu.py"""
    from riffusion import tc_ops

    def close(got, ref, tol=2e-3):
        err = (got.float() - ref).abs().max().item()
        assert err <= tol * ref.abs().max().item(), f"max err {err:.4e}"

    torch.manual_seed(W)
    B, H, C1, C2, Cout = 2, 64, 128, 64, 192
    x = (torch.randn(B, H, W, C1, device="cuda") * 0.5).half()
    x2 = (torch.randn(B, H, W, C2, device="cuda") * 0.5).half()
    for k, stride, cat in ((3, 1, False), (3, 2, False), (1, 1, False), (3, 1, True), (1, 1, True)):
        cin = C1 + (C2 if cat else 0)
        w = (torch.randn(Cout, cin, k, k, device="cuda") * cin ** -0.5 / k).half()
        bias = torch.randn(Cout, device="cuda").half()
        xin = torch.cat([x, x2], dim=3) if cat else x
        ref = torch.nn.functional.conv2d(xin.permute(0, 3, 1, 2).float(), w.float(), bias.float(), stride=stride,
                                         padding=1 if k == 3 else 0).permute(0, 2, 3, 1)
        got = tc_ops.conv2d(x, tc_ops.pack_conv_weight(w), x2=x2 if cat else None, bias=bias, stride=stride)
        assert got.shape == ref.shape
        close(got, ref)
    w = (torch.randn(Cout, C1, 3, 3, device="cuda") * C1 ** -0.5 / 3).half()
    bias = torch.randn(Cout, device="cuda").half()
    up = torch.nn.functional.interpolate(x.permute(0, 3, 1, 2).float(), scale_factor=2.0, mode="nearest")
    ref = torch.nn.functional.conv2d(up, w.float(), bias.float(), padding=1).permute(0, 2, 3, 1)
    got = tc_ops.conv2d_upsample2x(x, tc_ops.pack_upsample_weight(w), bias=bias)
    assert got.shape == ref.shape
    close(got, ref)


# ----------------------------------------------------------------------------------------------- G3
@torch.no_grad()
def test_sd15_unet_and_vae_at_64x96_latents(native_lib, vae_pair):
    """full-width SD-1.5 UNet, one CFG pair at 64x96 latents (a 768-wide clip), and the VAE decode of 64x96 latents to
    512x768, against the fp32 oracle at 1.15 x the fp16-storage floor + 1e-4"""
    from oracle import unet_emul as ue
    from oracle import unet_oracle as uo
    from riffusion.unet_b200 import UNetB200

    oracle = _round_params(uo.init_weights_(uo.UNet2DConditionOracle(), seed=0)).cuda().eval()
    ours = UNetB200(oracle.state_dict(), device="cuda")
    torch.manual_seed(96)
    x = torch.randn(2, 4, 64, 96, device="cuda").half()
    ctx = torch.randn(2, 77, 768, device="cuda").half()
    t = 741
    got = ours(x, t, encoder_hidden_states=ctx).sample
    assert got.shape == (2, 4, 64, 96)
    _check_vs_floor(got, oracle(x.float(), t, ctx.float()), ue.unet_forward(oracle, x, t, ctx), "UNet SD-1.5 64x96 B=2")
    del oracle, ours
    torch.cuda.empty_cache()
    voracle, vae = vae_pair
    z = (torch.randn(1, 4, 64, 96, device="cuda") * 4).half()
    img = vae.decode(z).sample
    assert img.shape == (1, 3, 512, 768)
    _check_vs_floor(img, voracle.decode(z.float()), ue.vae_decode(voracle, z), "VAE decode 64x96 latents")


# ----------------------------------------------------------------------------------------------- G4
@torch.no_grad()
@pytest.mark.parametrize("scheduler,steps", [("DPMSolverMultistepScheduler", 10), ("DPMSolverMultistepScheduler", 20),
                                             ("PNDMScheduler", 10)])
def test_txt2img_loop_matches_oracle_loop(small_unet, scheduler, steps):
    """txt2img (reduced-width UNet, 16x24 latents, injected latents and embeddings) against txt2img_loop on the fp32
    oracle; the floor is txt2img_loop_emul's distance to the fp32 loop"""
    from oracle import unet_oracle as uo
    from riffusion.riffusion_pipeline import RiffusionPipeline

    oracle, ours = small_unet
    pipe = RiffusionPipeline(vae=None, unet=ours, device="cuda")
    torch.manual_seed(steps)
    lat = torch.randn(1, 4, 16, 24, device="cuda").half()
    text = torch.randn(1, 77, 64, device="cuda").half()
    uncond = torch.randn(1, 77, 64, device="cuda").half()
    out = pipe.txt2img("", num_inference_steps=steps, width=192, height=128, scheduler=scheduler, output_type="latent",
                       text_embeddings=text, uncond_embeddings=uncond, latents=lat)
    mk = (lambda: DPMSolverMultistepOracle()) if scheduler.startswith("DPM") else uo.PNDMSchedulerOracle
    ref, n_ref = txt2img_loop(oracle, mk(), text.float(), uncond.float(), lat.float(), steps, 7.0)
    emul, n_emul = txt2img_loop_emul(oracle, mk(), text, uncond, lat, steps, 7.0)
    assert out["n_unet_evals"] == n_ref == n_emul == (steps if scheduler.startswith("DPM") else steps + 1)
    e, floor = rel_l2(out["latents_unscaled"], ref), rel_l2(emul, ref)
    print(f"txt2img {scheduler} {steps} steps: rel_l2 {e:.3e}, fp16-storage floor of the loop {floor:.3e}")
    assert e <= 1.3 * floor + 2e-4


# ----------------------------------------------------------------------------------------------- G5
@torch.no_grad()
def test_txt2img_graph_batch_and_seeds(small_unet):
    """graph replay equals the eager path bit for bit at 16x24 latents; three clips in one batch equal three single
    calls within the fp16 floor; clip i starts from the CUDA generator draw for seed + i"""
    from riffusion.riffusion_pipeline import RiffusionPipeline

    oracle, ours = small_unet
    pipe = RiffusionPipeline(vae=None, unet=ours, device="cuda")
    torch.manual_seed(5)
    text = torch.randn(1, 77, 64, device="cuda").half()
    uncond = torch.randn(1, 77, 64, device="cuda").half()
    kw = dict(num_inference_steps=8, width=192, height=128, output_type="latent", text_embeddings=text,
              uncond_embeddings=uncond)
    graphed = pipe.txt2img("", seed=3, num_clips=3, **kw)
    pipe.use_cuda_graph = False
    eager = pipe.txt2img("", seed=3, num_clips=3, **kw)
    pipe.use_cuda_graph = True
    assert torch.equal(graphed["latents_unscaled"], eager["latents_unscaled"])
    # batch-size dependent tiles / split-K make the single calls another equally valid fp16 evaluation: bound by the
    # loop's fp16-storage floor (clip 0), as far apart as two independent fp16 evaluations may be
    lat0 = torch.randn((1, 4, 16, 24), generator=torch.Generator("cuda").manual_seed(3), device="cuda", dtype=torch.float16)
    ref, _ = txt2img_loop(oracle, DPMSolverMultistepOracle(), text.float(), uncond.float(), lat0.float(), 8, 7.0)
    emul, _ = txt2img_loop_emul(oracle, DPMSolverMultistepOracle(), text, uncond, lat0, 8, 7.0)
    floor = rel_l2(emul, ref)
    draws = []
    for i in range(3):
        draws.append(torch.randn((1, 4, 16, 24), generator=torch.Generator("cuda").manual_seed(3 + i), device="cuda",
                                 dtype=torch.float16))
        single = pipe.txt2img("", seed=3 + i, num_clips=1, **kw)
        injected = pipe.txt2img("", num_clips=1, latents=draws[-1], **kw)
        assert torch.equal(single["latents_unscaled"], injected["latents_unscaled"])      # the draw for seed + i
        e = rel_l2(graphed["latents_unscaled"][i:i + 1], single["latents_unscaled"])
        print(f"clip {i}: batch of 3 vs single call {e:.3e} (fp16-storage floor of the loop {floor:.3e})")
        assert e <= 2 ** 0.5 * 1.3 * floor + 2e-4, (i, e, floor)
    batch_injected = pipe.txt2img("", num_clips=3, latents=torch.cat(draws), **kw)
    assert torch.equal(batch_injected["latents_unscaled"], graphed["latents_unscaled"])


# ----------------------------------------------------------------------------------------------- G6
def _stub_tokenizer():
    import sys
    from pathlib import Path

    sys.path.insert(0, str(Path(__file__).parent / "golden"))
    from prompt_stub import StubTokenizer

    return StubTokenizer()


def _t2a_pipe(vae):
    from riffusion import sd15_spec
    from riffusion.clip_b200 import ClipTextB200
    from riffusion.riffusion_pipeline import RiffusionPipeline
    from riffusion.unet_b200 import UNetB200

    c = SMALL["block_out_channels"]
    unet = UNetB200(sd15_spec.random_state_dict(sd15_spec.unet_spec(c, cross_attention_dim=768), 0), device="cuda",
                    block_out_channels=c, heads=4)
    return RiffusionPipeline(vae=vae, unet=unet, text_encoder=ClipTextB200.random_init(seed=2, layers=2),
                             tokenizer=_stub_tokenizer(), device="cuda")


@torch.no_grad()
@pytest.mark.parametrize("width,stereo", [(768, False), (512, True)])
def test_text_to_audio_end_to_end(vae_pair, width, stereo):
    """text_to_audio with the reduced UNet, the full VAE and a random-init CLIP; the device tail judged stage by stage:
    our latents -> fp32 oracle VAE -> uint8 vs our image; our uint8 image -> mel (R plane, or G and B for stereo) ->
    torchaudio inverse mel + Griffin-Lim with the same initial phases vs our waveform"""
    from oracle import audio_oracle as ao
    from oracle.torchaudio_ref import TorchaudioConverter
    from oracle.vae_oracle import u8_from_image_fp16
    from riffusion.spectrogram_params import SpectrogramParams

    oracle_vae, vae = vae_pair
    pipe = _t2a_pipe(vae)
    if stereo:
        params = SpectrogramParams(min_frequency=10, max_frequency=20000, stereo=True)
    else:
        params = SpectrogramParams(min_frequency=0, max_frequency=10000, stereo=False)
    C = 2 if stereo else 1
    torch.manual_seed(width)
    angles = torch.rand(C, 8821, width, dtype=torch.complex64, device="cuda")
    out = pipe.text_to_audio("church bells on sunday", params=params, negative_prompt="noise", seed=11,
                             num_inference_steps=6, width=width, init_angles=angles)
    assert out["images"].shape == (1, 512, width, 3) and out["images"].dtype == torch.uint8
    assert out["waveform"].shape == (1, C, 441 * (width - 1)) and torch.isfinite(out["waveform"]).all()
    assert out["n_unet_evals"] == 6
    u8 = out["images"].cpu().numpy()
    u8_ref = u8_from_image_fp16(oracle_vae.decode(out["latents"].float()).half())
    d = np.abs(u8.astype(np.int16) - u8_ref.astype(np.int16))
    print(f"text_to_audio {width} {'stereo' if stereo else 'mono'}: uint8 vs oracle VAE max {d.max()} LSB, "
          f"differing {100 * (d != 0).mean():.2f} %")
    assert d.max() <= 2 and (d != 0).mean() < 0.30 and (d > 1).mean() < 2e-3
    mel_ref = ao.spectrogram_from_image_array(u8[0], power=0.25, stereo=stereo, max_value=30e6)
    assert mel_ref.shape == (C, 512, width)
    ta = TorchaudioConverter(f_min=params.min_frequency, f_max=params.max_frequency)
    wave_ref = ta.waveform_from_mel_amplitudes(torch.from_numpy(mel_ref), angles.cpu())
    wave = out["waveform"][0].cpu()
    assert wave.shape == wave_ref.shape

    def nrms(a, b):
        return float((((a - b) / b.abs().amax(dim=-1, keepdim=True)) ** 2).mean().sqrt())

    rms = nrms(wave, wave_ref)
    print(f"text_to_audio {width}: waveform vs torchaudio on our uint8 image, normalised RMS {rms:.3e}")
    if rms >= 1e-4:
        # as in tests/test_parity_bench_gpu.py: Griffin-Lim amplifies fp32 rounding on a nearly flat random-weight image;
        # the fp64 oracle recurrence is the referee (channel 0), and we must be no further from it than twice torchaudio
        from riffusion.spectrogram_converter import mel_filterbank

        fb = mel_filterbank(8821, float(params.min_frequency), float(params.max_frequency), 512, 44100).numpy()
        o64 = torch.from_numpy(ao.waveform_from_mel_amplitudes(mel_ref[:1], fb, 17640, 441, ao.hann_window(4410).double().numpy(),
                                                               32, angles[:1].cpu().numpy())).float()
        e_ta, e_us = nrms(wave_ref[:1], o64), nrms(wave[:1], o64)
        print(f"text_to_audio {width}: vs the fp64 oracle recurrence: torchaudio fp32 {e_ta:.3e}, kernels {e_us:.3e}")
        assert e_us <= max(2 * e_ta, 2e-5)


# ----------------------------------------------------------------------------------------------- G7
def test_text_to_audio_cli(vae_pair, tmp_path, monkeypatch):
    """`text-to-audio` end to end with the checkpoint loader replaced by the reduced pipeline: a 768-wide clip lasts
    7.67 s, and the PNG's EXIF gives the same params to print-exif and image-to-audio"""
    import io
    from contextlib import redirect_stdout

    from PIL import Image

    from riffusion import cli
    from riffusion.riffusion_pipeline import RiffusionPipeline
    from riffusion.spectrogram_params import SpectrogramParams
    from riffusion.util.audio_util import AudioSegment

    _, vae = vae_pair
    pipe = _t2a_pipe(vae)
    monkeypatch.setattr(RiffusionPipeline, "load_checkpoint", classmethod(lambda cls, **kw: pipe))
    cli.main(["text-to-audio", "--prompt", "jazz with piano", "--audio", str(tmp_path / "out.wav"), "--image",
              str(tmp_path / "out.png"), "--width", "768", "--num-inference-steps", "4"])
    seg = AudioSegment.from_file(str(tmp_path / "out.wav"))
    assert seg.frame_rate == 44100 and seg.channels == 1
    assert abs(seg.duration_seconds - 7.67) < 0.01
    img = Image.open(tmp_path / "out.png")
    assert img.size == (768, 512)
    want = SpectrogramParams(min_frequency=0, max_frequency=10000, stereo=False)
    assert SpectrogramParams.from_exif(img.getexif()) == want
    buf = io.StringIO()
    with redirect_stdout(buf):
        cli.main(["print-exif", "--image", str(tmp_path / "out.png")])
    assert "NUM_FREQUENCIES" in buf.getvalue() and "10000" in buf.getvalue()
    cli.main(["image-to-audio", "--image", str(tmp_path / "out.png"), "--audio", str(tmp_path / "back.wav")])
    back = AudioSegment.from_file(str(tmp_path / "back.wav"))
    assert back.channels == 1 and abs(back.duration_seconds - 7.67) < 0.01
    cli.main(["text-to-audio", "--prompt", "jazz", "--audio", str(tmp_path / "s.wav"), "--image", str(tmp_path / "s.png"),
              "--num-clips", "2", "--seed", "5", "--use-20k", "--num-inference-steps", "3"])
    for s in (5, 6):
        seg = AudioSegment.from_file(str(tmp_path / f"s_{s}.wav"))
        assert seg.channels == 2 and abs(seg.duration_seconds - 5.11) < 0.01
        assert SpectrogramParams.from_exif(Image.open(tmp_path / f"s_{s}.png").getexif()).stereo
    torch.cuda.synchronize()
