"""Audio to audio on the H100: rf_resize_bicubic_u8 against Pillow bit for bit, img2img loops against the fp32 oracle loop
(tests/img2img_oracle.py; the start rule is unpinned for DPM-Solver++), graph replay / batching / generator draws,
audio_to_audio end to end judged stage by stage, and the `audio-to-audio` command.

Bars are those of tests/test_parity_bench_gpu.py: loops within 1.3 x the fp16-storage floor of the loop (+2e-4)."""
import numpy as np
import pytest
import torch
from PIL import Image

from img2img_oracle import img2img_loop, img2img_loop_emul
from test_audio_to_audio_cpu import RESIZES
from test_parity_bench_gpu import rel_l2
from test_text_to_audio_gpu import _no_tf32, _t2a_pipe, small_unet, vae_pair  # noqa: F401  (fixtures)
from txt2img_oracle import DPMSolverMultistepOracle

pytestmark = pytest.mark.gpu


# ----------------------------------------------------------------------------------------------- A1
@pytest.mark.parametrize("src,dst", RESIZES)
@pytest.mark.parametrize("channels", [1, 3])
def test_resize_kernel_is_pillow(native_lib, src, dst, channels):
    """three images per launch, bit-identical to PIL.Image.resize(BICUBIC); the fp16 output equals preprocess_image's
    torch expression on the same bytes"""
    from riffusion import tc_ops

    (w, h), (ow, oh) = src, dst
    rng = np.random.default_rng(w * 7 + h + channels)
    arr = rng.integers(0, 256, size=(3, h, w, channels), dtype=np.uint8)
    arr[0, : h // 2, : w // 2] = 255 * (arr[0, : h // 2, : w // 2] > 127)
    u8, f16 = tc_ops.resize_bicubic_u8(torch.from_numpy(arr).cuda(), ow, oh, want_f16=True)
    assert u8.shape == (3, oh, ow, channels) and f16.shape == (3, channels, oh, ow)
    got = u8.cpu().numpy()
    for i in range(3):
        im = Image.fromarray(arr[i, ..., 0] if channels == 1 else arr[i], "L" if channels == 1 else "RGB")
        want = np.asarray(im.resize((ow, oh), Image.BICUBIC))
        assert np.array_equal(got[i], want.reshape(oh, ow, channels)), i
    ref = 2.0 * torch.from_numpy(got.astype(np.float32) / 255.0) - 1.0
    assert torch.equal(f16.cpu(), ref.permute(0, 3, 1, 2).half())
    u8_only, none = tc_ops.resize_bicubic_u8(torch.from_numpy(arr).cuda(), ow, oh)
    assert none is None and torch.equal(u8_only, u8)


# ----------------------------------------------------------------------------------------------- A2
def _moments(n, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    mean = torch.randn((n, 4, 16, 24), generator=g, device="cuda").half()
    logvar = (torch.randn((n, 4, 16, 24), generator=g, device="cuda") * 0.2 - 0.5).half()
    return mean, logvar


def _draws(mean, logvar, seed):
    """what image i's generator (seeded with `seed`) draws: the fp32 posterior noise, then the fp16 img2img noise"""
    from riffusion.riffusion_pipeline import VAE_SCALE
    from riffusion.vae_b200 import _Posterior

    lats, noises = [], []
    for i in range(mean.shape[0]):
        g = torch.Generator(device="cuda").manual_seed(seed)
        lats.append(VAE_SCALE * _Posterior(mean[i:i + 1], logvar[i:i + 1]).sample(generator=g))
        noises.append(torch.randn(lats[-1].shape, generator=g, device="cuda", dtype=torch.float16))
    return torch.cat(lats), torch.cat(noises)


@torch.no_grad()
@pytest.mark.parametrize("scheduler", ["DPMSolverMultistepScheduler", "PNDMScheduler"])
def test_img2img_loop_matches_oracle_loop(small_unet, scheduler):
    """img2img (reduced-width UNet, 16x24 latents, injected moments and embeddings, 25 steps at strength 0.55) against
    img2img_loop on the fp32 oracle from the same generator draws; the floor is img2img_loop_emul's distance to it"""
    from oracle import unet_oracle as uo
    from riffusion.riffusion_pipeline import RiffusionPipeline

    oracle, ours = small_unet
    pipe = RiffusionPipeline(vae=None, unet=ours, device="cuda")
    torch.manual_seed(25)
    text = torch.randn(1, 77, 64, device="cuda").half()
    uncond = torch.randn(1, 77, 64, device="cuda").half()
    mean, logvar = _moments(1, 3)
    out = pipe.img2img("", None, strength=0.55, num_inference_steps=25, seed=11, scheduler=scheduler,
                       output_type="latent", text_embeddings=text, uncond_embeddings=uncond, moments=(mean, logvar))
    lat, noise = _draws(mean, logvar, 11)
    injected = pipe.img2img("", None, strength=0.55, num_inference_steps=25, seed=11, scheduler=scheduler,
                            output_type="latent", text_embeddings=text, uncond_embeddings=uncond, moments=(mean, logvar),
                            noise=noise)
    assert torch.equal(out["latents_unscaled"], injected["latents_unscaled"])         # the second draw is the noise
    mk = DPMSolverMultistepOracle if scheduler.startswith("DPM") else uo.PNDMSchedulerOracle
    ref, n_ref = img2img_loop(oracle, mk(), text.float(), uncond.float(), lat.float(), noise.float(), 25, 0.55, 7.0)
    emul, n_emul = img2img_loop_emul(oracle, mk(), text, uncond, lat, noise, 25, 0.55, 7.0)
    assert out["n_unet_evals"] == n_ref == n_emul == (13 if scheduler.startswith("DPM") else 14)
    e, floor = rel_l2(out["latents_unscaled"], ref), rel_l2(emul, ref)
    print(f"img2img {scheduler}: rel_l2 {e:.3e}, fp16-storage floor of the loop {floor:.3e}")
    assert e <= 1.3 * floor + 2e-4


@torch.no_grad()
def test_img2img_graph_batch_and_seeds(small_unet):
    """graph replay equals the eager path bit for bit; image i of a batch of 3 equals a single-image call within the fp16
    floor; every image's generator is seeded with the same seed"""
    from riffusion.riffusion_pipeline import RiffusionPipeline

    oracle, ours = small_unet
    pipe = RiffusionPipeline(vae=None, unet=ours, device="cuda")
    torch.manual_seed(6)
    text = torch.randn(1, 77, 64, device="cuda").half()
    uncond = torch.randn(1, 77, 64, device="cuda").half()
    mean, logvar = _moments(3, 4)
    kw = dict(strength=0.6, num_inference_steps=12, seed=2, output_type="latent", text_embeddings=text,
              uncond_embeddings=uncond)
    graphed = pipe.img2img("", None, moments=(mean, logvar), **kw)
    pipe.use_cuda_graph = False
    eager = pipe.img2img("", None, moments=(mean, logvar), **kw)
    pipe.use_cuda_graph = True
    assert torch.equal(graphed["latents_unscaled"], eager["latents_unscaled"])
    lat, noise = _draws(mean, logvar, 2)
    assert torch.equal(noise[0], noise[2])                                            # one seed for every image
    ref, _ = img2img_loop(oracle, DPMSolverMultistepOracle(), text.float(), uncond.float(), lat[:1].float(),
                          noise[:1].float(), 12, 0.6, 7.0)
    emul, _ = img2img_loop_emul(oracle, DPMSolverMultistepOracle(), text, uncond, lat[:1], noise[:1], 12, 0.6, 7.0)
    floor = rel_l2(emul, ref)
    for i in range(3):
        single = pipe.img2img("", None, moments=(mean[i:i + 1], logvar[i:i + 1]), **kw)
        e = rel_l2(graphed["latents_unscaled"][i:i + 1], single["latents_unscaled"])
        print(f"img2img image {i}: batch of 3 vs single call {e:.3e} (fp16-storage floor of the loop {floor:.3e})")
        assert e <= 2 ** 0.5 * 1.3 * floor + 2e-4, (i, e, floor)


# ----------------------------------------------------------------------------------------------- A3
def _track(stereo_source=True):
    from pathlib import Path

    from riffusion.util.audio_util import AudioSegment

    d = np.load(Path(__file__).parent / "golden" / "tired_traveler_clip2.npz")
    wav = np.tile(d["wav"], (2, 1))                                    # 11.36 s: clips at 0 and 4.8 s
    return AudioSegment(wav if stereo_source else wav[:, :1].copy(), int(d["rate"]))


def _params(stereo):
    from riffusion.spectrogram_params import SpectrogramParams

    if stereo:
        return SpectrogramParams(min_frequency=10, max_frequency=20000, stereo=True)
    return SpectrogramParams(min_frequency=0, max_frequency=10000, stereo=False)


@torch.no_grad()
@pytest.mark.parametrize("stereo", [False, True])
def test_audio_to_audio_end_to_end(vae_pair, stereo):
    """audio_to_audio with the reduced UNet, the full VAE and a random-init CLIP on a two-clip track, judged stage by
    stage: source images = spectrogram_image_from_audio of each clip byte for byte; both resizes = Pillow; the stitched
    track = stitch_segments over each riffed image's audio (host mel, the same Griffin-Lim phases, int16, filters);
    max_batch=1 gives the same result within the fp16 floor"""
    from riffusion import audio_to_audio as a2a
    from riffusion import tc_ops
    from riffusion.spectrogram_converter import SpectrogramConverter
    from riffusion.spectrogram_image_converter import SpectrogramImageConverter
    from riffusion.util import audio_util, image_util

    _, vae = vae_pair
    pipe = _t2a_pipe(vae)
    params = _params(stereo)
    C = 2 if stereo else 1
    track = _track()
    angles = torch.rand(2, C, 8821, 501, dtype=torch.complex64, device="cuda", generator=torch.Generator("cuda").manual_seed(1))
    kw = dict(params=params, num_inference_steps=10, seed=5, negative_prompt="noise", init_angles=angles)
    out = pipe.audio_to_audio(track, "church bells on sunday", **kw)
    assert np.allclose(out["clip_start_times"], [0.0, 4.8]) and out["n_unet_evals"] == [5]
    src, den, riffed = (out[k].cpu().numpy() for k in ("source_images", "denoised_images", "images"))
    assert src.shape == riffed.shape == (2, 512, 501, 3) and den.shape == (2, 512, 512, 3)
    clips = a2a.slice_audio_into_clips(track, out["clip_start_times"], 5.0)
    host = SpectrogramImageConverter(params, device="cuda")
    for i, clip in enumerate(clips):
        # the same mel amplitudes; the device quantiser (CUDA powf) agrees with numpy's except at truncation boundaries,
        # the bar tests/test_audio_gpu.py holds rf_mel_to_image to (mono clips come out byte for byte here)
        want = np.asarray(host.spectrogram_image_from_audio(clip))
        d = np.abs(src[i].astype(np.int16) - want.astype(np.int16))
        print(f"source image {i}: {int((d != 0).sum())} of {d.size} bytes differ, max {d.max()}")
        assert d.max() <= 1 and (d != 0).mean() < 1e-3, f"source image {i}"
        assert stereo or d.max() == 0
        assert np.array_equal(riffed[i], np.asarray(Image.fromarray(den[i]).resize((501, 512), Image.BICUBIC))), i
    up, _ = tc_ops.resize_bicubic_u8(out["source_images"], 512, 512)
    assert np.array_equal(up[1].cpu().numpy(), np.asarray(Image.fromarray(src[1]).resize((512, 512), Image.BICUBIC)))
    conv = SpectrogramConverter(params, device="cuda")
    segs = []
    for i in range(2):
        mel = image_util.spectrogram_from_image(Image.fromarray(riffed[i]), power=0.25, stereo=stereo, max_value=30e6)
        w = conv.waveform_from_mel_amplitudes(torch.from_numpy(mel).cuda(), angles[i]).cpu().numpy()
        segs.append(audio_util.apply_filters(audio_util.audio_from_waveform(w, 44100, normalize=True)))
    want = audio_util.stitch_segments(segs, crossfade_s=0.2)
    got = out["segment"]
    assert got.channels == C and abs(got.duration_seconds - 9.8) < 1e-3
    assert abs(got.duration_seconds - want.duration_seconds) < 1e-9
    a = np.asarray(got.get_array_of_samples(), dtype=np.float64)
    b = np.asarray(want.get_array_of_samples(), dtype=np.float64)
    nrms = float(np.sqrt(((a - b) ** 2).mean()) / np.abs(b).max())
    print(f"audio_to_audio {'stereo' if stereo else 'mono'}: stitched track vs host-side tail, normalised RMS {nrms:.3e}, "
          f"max |diff| {np.abs(a - b).max():.0f} LSB")
    assert nrms < 1e-3
    one = pipe.audio_to_audio(track, "church bells on sunday", max_batch=1, **kw)
    assert one["n_unet_evals"] == [5, 5]
    d = np.abs(one["images"].cpu().numpy().astype(np.int16) - riffed.astype(np.int16))
    print(f"audio_to_audio max_batch=1 vs 2: mean |diff| {d.mean():.4f} LSB, max {d.max()}")
    assert d.mean() < 0.25 and (d <= 1).mean() > 0.98


@torch.no_grad()
def test_audio_to_audio_interpolation_is_riffuse_batch(vae_pair):
    """with prompt_b, clip i is riffuse_batch's request i (alpha = linspace(0, 1, n)[i]) on the 32-stride source images"""
    from riffusion import tc_ops
    from riffusion.datatypes import InferenceInput, PromptInput

    _, vae = vae_pair
    pipe = _t2a_pipe(vae)
    track = _track()
    out = pipe.audio_to_audio(track, "church bells", prompt_b="jazz (piano:1.2)", seed=3, seed_b=8, denoising=0.5,
                              denoising_b=0.7, num_inference_steps=10, params=_params(False))
    up, _ = tc_ops.resize_bicubic_u8(out["source_images"], 512, 512)
    a = PromptInput(prompt="church bells", seed=3, denoising=0.5, guidance=7.0)
    b = PromptInput(prompt="jazz (piano:1.2)", seed=8, denoising=0.7, guidance=7.0)
    reqs = [InferenceInput(start=a, end=b, alpha=al, num_inference_steps=10) for al in (0.0, 1.0)]
    want = pipe.riffuse_batch(reqs, [Image.fromarray(im) for im in up.cpu().numpy()])
    for i in range(2):
        d = np.abs(out["denoised_images"][i].cpu().numpy().astype(np.int16) - np.asarray(want[i]).astype(np.int16))
        print(f"interpolation clip {i}: vs riffuse_batch mean |diff| {d.mean():.4f} LSB, max {d.max()}")
        assert d.mean() < 0.25 and (d <= 1).mean() > 0.98
    assert np.abs(np.asarray(want[0]).astype(np.int16) - np.asarray(want[1]).astype(np.int16)).mean() > 0.5


def test_audio_to_audio_cli(vae_pair, tmp_path, monkeypatch):
    """`audio-to-audio` end to end with the checkpoint loader replaced by the reduced pipeline"""
    from riffusion import cli
    from riffusion.riffusion_pipeline import RiffusionPipeline
    from riffusion.spectrogram_params import SpectrogramParams
    from riffusion.util.audio_util import AudioSegment

    _, vae = vae_pair
    pipe = _t2a_pipe(vae)
    monkeypatch.setattr(RiffusionPipeline, "load_checkpoint", classmethod(lambda cls, **kw: pipe))
    _track().export(str(tmp_path / "in.wav"), format="wav")
    cli.main(["audio-to-audio", "--audio", str(tmp_path / "in.wav"), "--output", str(tmp_path / "out.wav"), "--prompt",
              "jazz with piano", "--image-dir", str(tmp_path / "img"), "--num-inference-steps", "6", "--use-20k"])
    seg = AudioSegment.from_file(str(tmp_path / "out.wav"))
    assert seg.frame_rate == 44100 and seg.channels == 2 and abs(seg.duration_seconds - 9.8) < 1e-3
    want = SpectrogramParams(min_frequency=10, max_frequency=20000, stereo=True)
    for i in range(2):
        for kind in ("source", "riffed"):
            img = Image.open(tmp_path / "img" / f"clip_{i}_{kind}.png")
            assert img.size == (501, 512) and SpectrogramParams.from_exif(img.getexif()) == want
    torch.cuda.synchronize()
