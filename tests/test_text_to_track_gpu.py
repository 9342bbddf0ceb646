"""Long tracks on the H100: the window gather and merge kernels against torch and fp64, the windowed loop against
txt2img where the two must agree bit for bit (one window; windows without overlap), against the fp32 windowed oracle
loop with overlap, graph replay, the query-chunked VAE attention, text_to_track end to end at more than 3000 frames,
and the `text-to-track` command.

Bars are those of tests/test_text_to_audio_gpu.py: whole-network outputs within 1.15 x the fp16-storage floor (+1e-4)
of the fp32 oracle, loops within 1.3 x the floor of the loop (+2e-4)."""
import numpy as np
import pytest
import torch

import track_oracle as to
from test_parity_bench_gpu import _check_vs_floor, _round_params, rel_l2
from txt2img_oracle import DPMSolverMultistepOracle

pytestmark = pytest.mark.gpu

SMALL = dict(block_out_channels=(64, 128, 128, 128), heads=4, cross_attention_dim=64)
SCHEDULERS = ["DPMSolverMultistepScheduler", "PNDMScheduler", "DDIMScheduler", "EulerAncestralDiscreteScheduler"]


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


def _embeddings(seed, rows=1):
    g = torch.Generator(device="cuda").manual_seed(seed)
    text = torch.randn(rows, 77, 64, generator=g, device="cuda").half()
    uncond = torch.randn(1, 77, 64, generator=g, device="cuda").half()
    return text, uncond


# ----------------------------------------------------------------------------------------------- kernels
@pytest.mark.parametrize("n", [1, 2, 5])
@pytest.mark.parametrize("s_div", [1, 2, 4, 8])
@pytest.mark.parametrize("groups", [2, 6])
def test_gather_and_merge_kernels(native_lib, n, s_div, groups):
    """gather equals torch indexing bit for bit; merge is within one fp16 ulp of the fp64 sum of the covering windows
    (Ww = 64 latent columns, s = Ww, Ww/2, Ww/4 and 8; 2 groups: one track without CFG pairs, 6: three CFG tracks)"""
    from riffusion import window_ops

    Ww = 64
    s = Ww // s_div
    win = window_ops.Windows.make(Ww, s, n, "cuda")
    torch.manual_seed(n * 100 + s_div * 10 + groups)
    canvas = (torch.randn(groups, 4, 16, win.canvas, device="cuda") * 3).half()
    got = window_ops.window_gather(canvas, win)
    assert torch.equal(got, to.gather(canvas, Ww, s, n))
    windows = (torch.randn(groups * n, 4, 16, Ww, device="cuda") * 3).half()
    merged = window_ops.window_merge(windows, win)
    ref = to.merge_f64(windows, Ww, s, n)
    ulp = np.finfo(np.float16).eps * np.maximum(np.abs(ref), 2.0 ** -14)
    assert np.all(np.abs(merged.double().cpu().numpy() - ref) <= ulp)
    # a column covered by one window is that window's value, bit for bit
    if s == Ww:
        assert torch.equal(merged, torch.cat(windows.view(groups, n, 4, 16, Ww).unbind(1), dim=-1))
    assert torch.equal(merged[..., :s], windows.view(groups, n, 4, 16, Ww)[:, 0, ..., :s])


# ----------------------------------------------------------------------------------------------- loops
@torch.no_grad()
@pytest.mark.parametrize("scheduler", SCHEDULERS)
def test_one_window_track_is_txt2img(small_unet, scheduler):
    """a track of one window (width == window_width) is txt2img at that width, bit for bit, two tracks at once"""
    from riffusion.riffusion_pipeline import RiffusionPipeline

    _, ours = small_unet
    pipe = RiffusionPipeline(vae=None, unet=ours, device="cuda")
    text, uncond = _embeddings(1)
    kw = dict(num_inference_steps=6, height=128, scheduler=scheduler, output_type="latent", text_embeddings=text,
              uncond_embeddings=uncond, seed=9)
    track = pipe.txt2img_track("", width=256, window_width=256, stride=128, num_tracks=2, **kw)
    ref = pipe.txt2img("", width=256, num_clips=2, **kw)
    assert track["windows"] == [0] and track["loops"] == [[0, 1]]
    assert track["n_unet_evals"] == ref["n_unet_evals"]
    assert torch.equal(track["latents_unscaled"], ref["latents_unscaled"])


@torch.no_grad()
@pytest.mark.parametrize("scheduler", SCHEDULERS)
def test_abutting_windows_are_txt2img_of_the_crops(small_unet, scheduler):
    """stride == window_width: the canvas is txt2img of its crops stacked as one batch (injected latents and step noise,
    one prompt per window), bit for bit"""
    from riffusion.riffusion_pipeline import RiffusionPipeline

    _, ours = small_unet
    pipe = RiffusionPipeline(vae=None, unet=ours, device="cuda")
    n, T_, steps = 3, 2, 5
    text, uncond = _embeddings(2, rows=n)
    torch.manual_seed(3)
    lat = torch.randn(T_, 4, 16, 32 * n, device="cuda").half()
    noise = torch.randn(steps, T_, 4, 16, 32 * n, device="cuda").half() if scheduler.startswith("Euler") else None
    kw = dict(num_inference_steps=steps, height=128, scheduler=scheduler, output_type="latent", uncond_embeddings=uncond)
    track = pipe.txt2img_track("", width=256 * n, window_width=256, stride=256, num_tracks=T_, text_embeddings=text,
                               latents=lat, step_noise=noise, **kw)
    crops = to.gather(lat, 32, 32, n)
    crop_noise = None if noise is None else torch.stack([to.gather(z, 32, 32, n) for z in noise])
    ref = pipe.txt2img("", width=256, num_clips=T_ * n, text_embeddings=text.repeat(T_, 1, 1), latents=crops,
                       step_noise=crop_noise, **kw)
    canvas = torch.cat([ref["latents_unscaled"].view(T_, n, 4, 16, 32)[:, k] for k in range(n)], dim=-1)
    assert torch.equal(track["latents_unscaled"], canvas)


@torch.no_grad()
@pytest.mark.parametrize("s,prompts", [(16, 1), (8, 1), (16, 2)])
def test_overlapping_track_matches_oracle_loop(small_unet, s, prompts):
    """overlapping windows (s = Ww/2 and Ww/4 latent columns) on the reduced UNet at height 128 against the fp32 windowed
    oracle loop, at 1.3 x the floor of its fp16-storage emulation + 2e-4; `prompts` 2: the windows' text switches
    halfway along the track"""
    from riffusion.riffusion_pipeline import RiffusionPipeline

    oracle, ours = small_unet
    pipe = RiffusionPipeline(vae=None, unet=ours, device="cuda")
    Ww, n, steps = 32, 3, 10
    text, uncond = _embeddings(4, rows=prompts)
    texts = text if prompts == 1 else torch.cat([text[:1], text[:1], text[1:]])
    torch.manual_seed(s + prompts)
    lat = torch.randn(1, 4, 16, Ww + (n - 1) * s, device="cuda").half()
    out = pipe.txt2img_track("", width=8 * lat.shape[-1], height=128, window_width=8 * Ww, stride=8 * s,
                             num_inference_steps=steps, output_type="latent", text_embeddings=texts,
                             uncond_embeddings=uncond, latents=lat)
    assert out["windows"] == [0, 8 * s, 16 * s]
    texts_n = texts.expand(n, -1, -1)
    ref, n_ref = to.track_loop(oracle, DPMSolverMultistepOracle(), texts_n.float(), uncond.float(), lat.float(), steps,
                               7.0, Ww, s)
    emul, n_emul = to.track_loop_emul(oracle, DPMSolverMultistepOracle(), texts_n, uncond, lat, steps, 7.0, Ww, s)
    assert out["n_unet_evals"] == n_ref == n_emul == steps
    e, floor = rel_l2(out["latents_unscaled"], ref), rel_l2(emul, ref)
    print(f"track s={s} prompts={prompts}: rel_l2 {e:.3e}, fp16-storage floor of the loop {floor:.3e}")
    assert e <= 1.3 * floor + 2e-4


@torch.no_grad()
def test_track_graph_replay_equals_eager(small_unet):
    from riffusion.riffusion_pipeline import RiffusionPipeline

    _, ours = small_unet
    pipe = RiffusionPipeline(vae=None, unet=ours, device="cuda")
    text, uncond = _embeddings(5, rows=3)
    kw = dict(width=512, height=128, window_width=256, stride=128, num_tracks=3, max_batch=6, num_inference_steps=5,
              output_type="latent", text_embeddings=text, uncond_embeddings=uncond, seed=2)
    graphed = pipe.txt2img_track("", **kw)
    pipe.use_cuda_graph = False
    eager = pipe.txt2img_track("", **kw)
    assert graphed["loops"] == eager["loops"] == [[0, 1], [2]]
    assert torch.equal(graphed["latents_unscaled"], eager["latents_unscaled"])


# ----------------------------------------------------------------------------------------------- VAE and audio
@torch.no_grad()
def test_query_chunked_vae_attention(vae_pair):
    """the VAE decode with its mid-block attention split into query chunks (forced by a small max_score_bytes) against
    the fp32 oracle at the floor of tests/test_text_to_audio_gpu.py, and against the unchunked decode"""
    from oracle import unet_emul as ue

    voracle, vae = vae_pair
    torch.manual_seed(12)
    z = (torch.randn(1, 4, 64, 96, device="cuda") * 4).half()
    whole = vae.decode(z).sample
    saved = vae.max_score_bytes
    try:
        vae.max_score_bytes = 6144 * 640 * 2          # 640 of 6144 query rows per launch: ten chunks, the last short
        chunked = vae.decode(z).sample
    finally:
        vae.max_score_bytes = saved
    print(f"chunked vs unchunked VAE decode: rel_l2 {rel_l2(chunked, whole):.3e}")
    _check_vs_floor(chunked, voracle.decode(z.float()), ue.vae_decode(voracle, z), "VAE decode, query-chunked attention")


def _track_pipe(vae):
    from test_text_to_audio_gpu import _t2a_pipe

    return _t2a_pipe(vae)


@torch.no_grad()
def test_text_to_track_end_to_end(vae_pair):
    """text_to_track of 30 s (3001 frames on a 3072-column canvas, 11 windows) with two prompt spans, the reduced UNet,
    the full VAE and a random-init CLIP: our latents -> fp32 oracle VAE -> uint8 vs our image; our uint8 image ->
    torchaudio inverse mel + Griffin-Lim with the same initial phases vs our waveform; exactly round(30 sr) samples"""
    from oracle import audio_oracle as ao
    from oracle.torchaudio_ref import TorchaudioConverter
    from oracle.vae_oracle import u8_from_image_fp16

    oracle_vae, vae = vae_pair
    pipe = _track_pipe(vae)
    torch.manual_seed(30)
    angles = torch.rand(1, 1, 8821, 3072, dtype=torch.complex64, device="cuda")
    out = pipe.text_to_track([(0, "lo-fi piano"), (15, "jazz with drums")], duration_s=30.0, num_inference_steps=3,
                             seed=4, init_angles=angles)
    assert len(out["windows"]) == 11 and out["loops"] == [[0]] and out["n_unet_evals"] == 3
    assert [w["prompt"] for w in out["windows"]] == ["lo-fi piano"] * 5 + ["jazz with drums"] * 6
    assert out["images"].shape == (1, 512, 3072, 3)
    assert out["waveform"].shape == (1, 1, 30 * 44100) and torch.isfinite(out["waveform"]).all()
    u8 = out["images"].cpu().numpy()
    u8_ref = u8_from_image_fp16(oracle_vae.decode(out["latents"].float()).half())
    d = np.abs(u8.astype(np.int16) - u8_ref.astype(np.int16))
    print(f"text_to_track: uint8 vs oracle VAE max {d.max()} LSB, differing {100 * (d != 0).mean():.2f} %")
    assert d.max() <= 2 and (d != 0).mean() < 0.30 and (d > 1).mean() < 2e-3
    del u8_ref
    torch.cuda.empty_cache()
    mel_ref = ao.spectrogram_from_image_array(u8[0], power=0.25, stereo=False, max_value=30e6)
    wave_ref = TorchaudioConverter(f_min=0, f_max=10000).waveform_from_mel_amplitudes(torch.from_numpy(mel_ref),
                                                                                      angles[0].cpu())
    assert wave_ref.shape == (1, 441 * 3071)
    wave = out["waveform"][0].cpu()
    wave_ref = wave_ref[..., :wave.shape[-1]]
    rms = float((((wave - wave_ref) / wave_ref.abs().amax(dim=-1, keepdim=True)) ** 2).mean().sqrt())
    print(f"text_to_track: waveform vs torchaudio on our uint8 image (3072 frames), normalised RMS {rms:.3e}")
    assert rms < 1e-4


def test_text_to_track_cli(vae_pair, tmp_path, monkeypatch):
    """`text-to-track` with the checkpoint loader replaced by the reduced pipeline: a 6 s track lasts exactly 6 s, and
    its PNG's EXIF gives image-to-audio the same params"""
    from PIL import Image

    from riffusion import cli
    from riffusion.riffusion_pipeline import RiffusionPipeline
    from riffusion.spectrogram_params import SpectrogramParams
    from riffusion.util.audio_util import AudioSegment

    _, vae = vae_pair
    pipe = _track_pipe(vae)
    monkeypatch.setattr(RiffusionPipeline, "load_checkpoint", classmethod(lambda cls, **kw: pipe))
    cli.main(["text-to-track", "--prompt", "lo-fi piano", "--prompt-changes", "3:hard rock", "--audio",
              str(tmp_path / "out.wav"), "--image", str(tmp_path / "out.png"), "--duration-s", "6",
              "--num-inference-steps", "3"])
    seg = AudioSegment.from_file(str(tmp_path / "out.wav"))
    assert seg.frame_rate == 44100 and seg.channels == 1 and len(seg.get_array_of_samples()) == 6 * 44100
    img = Image.open(tmp_path / "out.png")
    assert img.size == (768, 512)              # 601 frames -> 512 + 256
    assert SpectrogramParams.from_exif(img.getexif()) == SpectrogramParams(min_frequency=0, max_frequency=10000,
                                                                           stereo=False)
    cli.main(["image-to-audio", "--image", str(tmp_path / "out.png"), "--audio", str(tmp_path / "back.wav")])
    back = AudioSegment.from_file(str(tmp_path / "back.wav"))
    assert back.channels == 1 and abs(back.duration_seconds - 441 * 767 / 44100) < 0.01
    torch.cuda.synchronize()
