"""Audio to audio on the host: the clip bookkeeping against the reference's expressions, the bicubic resize's tap tables
applied with the kernel's integer arithmetic against Pillow, the img2img start rule (unpinned for DPM-Solver++: it
restates diffusers from memory) and the control flow of RiffusionPipeline.img2img with the device steps replaced by
their torch definitions, and the `audio-to-audio` command."""
import importlib.util
import sys
import types
from pathlib import Path

import numpy as np
import pytest
import torch
from PIL import Image

ROOT = Path(__file__).resolve().parents[1]


def _track(seconds: float, channels: int = 1, rate: int = 44100, seed: int = 0):
    from riffusion.util.audio_util import AudioSegment

    rng = np.random.default_rng(seed)
    return AudioSegment(rng.integers(-8000, 8000, size=(int(seconds * rate), channels)).astype(np.int16), rate)


# ----------------------------------------------------------------------------------------------- clips
def test_clip_start_times_cuts_and_stitched_length():
    """a 20 s request on a 60 s track: starts 0, 4.8, 9.6, 14.4 s cut at [0, 4800, 9600, 14399] ms (14.4 * 1000 =
    14399.999...), 220 500 samples each, stitched with a 0.2 s crossfade to 4 * 5.0 - 3 * 0.2 = 19.4 s"""
    from riffusion import audio_to_audio as a2a
    from riffusion.util import audio_util

    track = _track(60.0)
    starts = a2a.clip_start_times(track.duration_seconds)
    assert np.allclose(starts, [0.0, 4.8, 9.6, 14.4])
    assert [int(s * 1000) for s in starts] == [0, 4800, 9600, 14399]
    clips = a2a.slice_audio_into_clips(track, starts, 5.0)
    samples = track.get_array_of_samples()
    for s, c in zip(starts, clips):
        assert len(c.get_array_of_samples()) == 220500
        first = int(int(s * 1000) * 44100 / 1000.0)
        assert np.array_equal(np.asarray(c.get_array_of_samples()), np.asarray(samples)[first:first + 220500])
    assert a2a.clip_frames(5.0, 44100, 441) == 501 and a2a.stride_32_size(501, 512) == (512, 512)
    stitched = audio_util.stitch_segments(clips, crossfade_s=0.2)
    assert abs(stitched.duration_seconds - 19.4) < 1e-9
    # the duration is cut to what the track holds after the start time; the last start stays one clip short of the end
    assert np.allclose(a2a.clip_start_times(11.0), [0.0, 4.8])
    assert np.allclose(a2a.clip_start_times(60.0, start_time_s=50.0), [50.0, 54.8])
    assert len(a2a.clip_start_times(5.0)) == 0


def test_last_clip_is_padded_with_silence():
    """a clip list whose last clip runs past the end of the track is padded with silence (audio_to_audio.py:408-412)"""
    from riffusion import audio_to_audio as a2a

    track = _track(7.0)
    clips = a2a.slice_audio_into_clips(track, [0.0, 4.0], 5.0)
    assert abs(clips[0].duration_seconds - 5.0) < 1e-9
    assert abs(clips[1].duration_seconds - 5.0) < 1e-3
    tail = np.asarray(clips[1].get_array_of_samples())[3 * 44100 + 10:]
    assert len(tail) > 0 and not tail.any()


@pytest.mark.parametrize("clip_s,ok", [(3.0, True), (4.0, False), (5.0, True), (6.0, False), (7.0, True), (8.0, True),
                                       (9.0, False), (10.0, True)])
def test_clip_durations_the_denoiser_takes(clip_s, ok):
    from riffusion import audio_to_audio as a2a

    w, h = a2a.stride_32_size(a2a.clip_frames(clip_s, 44100, 441), 512)
    if ok:
        a2a.check_denoising_size(w, h, clip_s)
    else:
        with pytest.raises(ValueError, match="3, 5, 7, 8 and 10 s work and 4, 6 and 9 s do not"):
            a2a.check_denoising_size(w, h, clip_s)


def test_audio_to_audio_rejects_before_device_work():
    """a track shorter than one clip (the reference's arange is empty and its stitch would fail) and a clip duration
    whose image width is not a multiple of 64 raise ValueError before anything runs on a device"""
    from riffusion.riffusion_pipeline import RiffusionPipeline

    pipe = RiffusionPipeline(vae=None, unet=None, device="cpu")
    with pytest.raises(ValueError, match="shorter than one clip"):
        pipe.audio_to_audio(_track(4.0), "jazz")
    with pytest.raises(ValueError, match="shorter than one clip"):
        pipe.audio_to_audio(_track(30.0), "jazz", start_time_s=26.0)
    with pytest.raises(ValueError, match="multiples of 64"):
        pipe.audio_to_audio(_track(30.0), "jazz", clip_duration_s=4.0)
    with pytest.raises(ValueError, match="max_batch"):
        pipe.audio_to_audio(_track(30.0), "jazz", max_batch=0)


# ----------------------------------------------------------------------------------------------- resize tables
def apply_table(arr: np.ndarray, table, axis: int) -> np.ndarray:
    """one pass of rf_resize_bicubic_u8 in numpy: (1 << 21) + sum u8 * tap in integers, >> 22, clamped to 0..255"""
    first, count, taps = table
    a = np.moveaxis(arr.astype(np.int64), axis, 0)
    out = np.empty((len(first),) + a.shape[1:], dtype=np.int64)
    for o in range(len(first)):
        acc = np.full(a.shape[1:], 1 << 21, dtype=np.int64)
        for j in range(count[o]):
            acc += a[first[o] + j] * int(taps[o, j])
        out[o] = np.where(acc >= 1 << 30, 255, np.where(acc <= 0, 0, acc >> 22))
    return np.moveaxis(out, 0, axis).astype(np.uint8)


RESIZES = [((501, 512), (512, 512)), ((512, 512), (501, 512)), ((568, 40), (576, 48)), ((576, 37), (568, 40)),
           ((300, 97), (97, 300)), ((97, 300), (300, 97)), ((1, 5), (13, 1)), ((13, 1), (1, 9)), ((7, 6), (7, 6)),
           ((64, 3), (2, 3))]


@pytest.mark.parametrize("src,dst", RESIZES)
@pytest.mark.parametrize("mode", ["L", "RGB"])
def test_resize_tables_reproduce_pillow(native_lib, src, dst, mode):
    """the host tap tables (fp64, rounded to 22 fractional bits) applied horizontally first with the kernel's integer
    arithmetic reproduce PIL.Image.resize(BICUBIC) on every pixel, up and down, including 1 -> n and n -> 1"""
    from riffusion import tc_ops

    (w, h), (ow, oh) = src, dst
    rng = np.random.default_rng(w * 1000 + h)
    arr = rng.integers(0, 256, size=(h, w) + ((3,) if mode == "RGB" else ()), dtype=np.uint8)
    arr[: h // 2, : w // 2] = 255 * (arr[: h // 2, : w // 2] > 127)         # hard edges: the negative lobes clamp
    want = np.asarray(Image.fromarray(arr, mode).resize((ow, oh), Image.BICUBIC))
    got = arr
    if ow != w:
        got = apply_table(got, tc_ops.resize_bicubic_table(w, ow), 1)
    if oh != h:
        got = apply_table(got, tc_ops.resize_bicubic_table(h, oh), 0)
    assert np.array_equal(got, want)


def test_resize_table_shape_and_identity(native_lib):
    from riffusion import tc_ops

    first, count, taps = tc_ops.resize_bicubic_table(501, 512)
    assert taps.shape == (512, 5) and count.max() <= 5 and first.min() == 0 and (first + count).max() == 501
    first, count, taps = tc_ops.resize_bicubic_table(512, 501)
    assert taps.shape == (501, 7)
    assert np.all(np.abs(taps.sum(axis=1) - (1 << 22)) <= 4)
    first, count, taps = tc_ops.resize_bicubic_table(9, 9)          # equal sizes: the taps are the identity
    rows = np.zeros((9, 9), dtype=np.int64)
    for o in range(9):
        rows[o, first[o]:first[o] + count[o]] = taps[o, :count[o]]
    assert np.array_equal(rows, np.eye(9, dtype=np.int64) << 22)
    with pytest.raises(ValueError):
        tc_ops.resize_bicubic_table(0, 5)


# ----------------------------------------------------------------------------------------------- img2img start rule
@pytest.mark.parametrize("steps,strength,evals_dpm,evals_pndm", [(25, 0.55, 13, 14), (25, 0.4, 10, 11), (25, 1.0, 25, 25),
                                                                  (50, 0.75, 37, 38), (10, 0.5, 5, 6), (20, 0.05, 1, 2)])
def test_img2img_start_rule(steps, strength, evals_dpm, evals_pndm):
    """evaluation counts and start timesteps of both schedulers (unpinned for DPM-Solver++); for PNDM the start
    timestep is interpolate_img2img's timesteps[-init_timestep] and the count its len(timesteps[t_start:])"""
    from riffusion.riffusion_pipeline import RiffusionPipeline
    from riffusion.scheduler_b200 import make_scheduler

    for name, want in (("DPMSolverMultistepScheduler", evals_dpm), ("PNDMScheduler", evals_pndm)):
        s = make_scheduler(name)
        s.set_timesteps(steps)
        t_start = RiffusionPipeline.img2img_start(s, steps, strength)
        assert len(s.timesteps[t_start:]) == want, name
        offset = s.config.get("steps_offset", 0)
        init_timestep = min(int(steps * strength) + offset, steps)
        assert int(s.timesteps[t_start]) == int(s.timesteps[-init_timestep]), name
    s = make_scheduler("DPMSolverMultistepScheduler")
    s.set_timesteps(25)
    assert RiffusionPipeline.img2img_start(s, 25, 0.55) == 12 and int(s.timesteps[12]) == 519


@pytest.mark.parametrize("steps,strength", [(25, 0.55), (10, 0.5), (14, 0.6)])
def test_dpm_plan_mid_schedule(steps, strength):
    """a DPM-Solver++ loop that starts mid-schedule is first order on its first step and second order after; the last
    step is first order only when the whole schedule has fewer than 15 steps"""
    from riffusion.riffusion_pipeline import RiffusionPipeline
    from riffusion.scheduler_b200 import DPMSolverMultistepSchedulerB200

    s = DPMSolverMultistepSchedulerB200()
    s.set_timesteps(steps)
    ts = s.timesteps.tolist()
    t_start = RiffusionPipeline.img2img_start(s, steps, strength)
    orders = []
    for i, t in enumerate(ts[t_start:]):
        order, coefs = s.plan(t)
        orders.append(order)
        if order == 2:          # the midpoint term uses the step actually run before this one
            s1 = ts[t_start + i - 1]
            nxt = 0 if t_start + i == len(ts) - 1 else ts[t_start + i + 1]
            h = s.lambda_t[nxt] - s.lambda_t[t]
            assert coefs[4] == pytest.approx(0.5 * coefs[3] * h / (s.lambda_t[t] - s.lambda_t[s1]), rel=1e-12)
        s.lower_order_nums = min(s.lower_order_nums + 1, 2)
    assert orders[0] == 1 and all(o == 2 for o in orders[1:-1])
    assert orders[-1] == (1 if steps < 15 else 2)


# ----------------------------------------------------------------------------------------------- img2img control flow
class _RecordingUNet:
    def __init__(self):
        self.inputs, self.timesteps = [], []

    def __call__(self, x, t, encoder_hidden_states=None, **kw):
        self.inputs.append(x.clone())
        self.timesteps.append(t)
        out = 0.3 * torch.tanh(x.float()) + 0.002 * (t / 1000.0) + \
            0.05 * encoder_hidden_states.float().mean(dim=(1, 2))[:, None, None, None]
        return types.SimpleNamespace(sample=out.to(torch.float16))


def _pipe(monkeypatch, scheduler=None):
    from test_text_to_audio_cpu import _fake_dpm_step, _fake_pndm_step

    from riffusion import tc_ops
    from riffusion.riffusion_pipeline import RiffusionPipeline

    def dpm(eps_pair, guidance, sample, m1, coefs):
        x0, prev = _fake_dpm_step(eps_pair.float(), guidance, sample.float(), None if m1 is None else m1.float(), coefs)
        return x0.half(), prev.half()

    def axpby(x, noise, a, b, mask=None, z=None):
        return (a * x.float() + b * noise.float()).half()

    monkeypatch.setattr(tc_ops, "cfg_dpmpp_step", dpm)
    monkeypatch.setattr(tc_ops, "cfg_pndm_step", _fake_pndm_step)
    monkeypatch.setattr(tc_ops, "axpby", axpby)
    unet = _RecordingUNet()
    pipe = RiffusionPipeline(vae=None, unet=unet, scheduler=scheduler, device="cpu")
    pipe.use_cuda_graph = False
    return pipe, unet


def test_img2img_control_flow_and_draws(monkeypatch):
    """img2img with injected moments: clip i's generator (seeded with `seed` for every clip) draws the fp32 posterior
    noise, then the fp16 img2img noise; noise is added at timesteps[t_start]; one CFG evaluation per remaining timestep"""
    from riffusion.riffusion_pipeline import VAE_SCALE
    from riffusion.scheduler_b200 import make_scheduler

    pipe, unet = _pipe(monkeypatch)
    torch.manual_seed(3)
    mean = torch.randn(3, 4, 8, 8).half()
    logvar = (torch.randn(3, 4, 8, 8) * 0.5 - 2).half()
    text, uncond = torch.randn(1, 77, 16).half(), torch.randn(1, 77, 16).half()
    for sched, n_want in (("DPMSolverMultistepScheduler", 13), ("PNDMScheduler", 14)):
        unet.inputs.clear()
        unet.timesteps.clear()
        out = pipe.img2img("", None, strength=0.55, num_inference_steps=25, seed=9, scheduler=sched, output_type="latent",
                           text_embeddings=text, uncond_embeddings=uncond, moments=(mean, logvar))
        assert out["n_unet_evals"] == n_want == len(unet.inputs) and out["t_start"] == 12
        s = make_scheduler(sched)
        s.set_timesteps(25)
        assert unet.timesteps == [int(t) for t in s.timesteps[12:]]
        first = unet.inputs[0]
        assert first.shape == (6, 4, 8, 8)
        a = float(s.alphas_cumprod[int(s.timesteps[12])])
        for i in range(3):
            g = torch.Generator().manual_seed(9)
            post = torch.randn((1, 4, 8, 8), generator=g)                                    # fp32 posterior draw
            std = torch.exp(0.5 * torch.clamp(logvar[i:i + 1], -30.0, 20.0))
            lat = VAE_SCALE * (mean[i:i + 1].float() + std.float() * post).half()
            noise = torch.randn((1, 4, 8, 8), generator=g, dtype=torch.float16)              # then the fp16 noise
            want = (a ** 0.5 * lat.float() + (1 - a) ** 0.5 * noise.float()).half()
            assert torch.equal(first[i:i + 1], want) and torch.equal(first[3 + i:4 + i], want)
    with pytest.raises(ValueError, match="noise must be"):
        pipe.img2img("", None, moments=(mean, logvar), noise=torch.zeros(2, 4, 8, 8), text_embeddings=text,
                     uncond_embeddings=uncond, output_type="latent")
    with pytest.raises(ValueError, match="DPMSolverMultistepScheduler, PNDMScheduler"):
        pipe.img2img("", None, moments=(mean, logvar), scheduler="LMSDiscreteScheduler", text_embeddings=text,
                     uncond_embeddings=uncond)


def test_zero_step_edge_of_both_img2img_entry_points(monkeypatch):
    """when the start rule leaves no timestep to run, interpolate_img2img returns the latents noised at
    timesteps[-init_timestep] (PNDM at 1 step: t = 1; DPM-Solver++ at 25 steps and strength 0.02: init_timestep = 0, so
    timesteps[0] = 999) and img2img returns the clean latents; neither evaluates the UNet"""
    from riffusion.riffusion_pipeline import VAE_SCALE
    from riffusion.scheduler_b200 import DPMSolverMultistepSchedulerB200, PNDMSchedulerB200

    torch.manual_seed(6)
    lat, noise = torch.randn(2, 4, 8, 8).half(), torch.randn(2, 4, 8, 8).half()
    mean, logvar = torch.randn(2, 4, 8, 8).half(), (torch.randn(2, 4, 8, 8) * 0.5 - 2).half()
    text, uncond = torch.randn(2, 77, 16).half(), torch.randn(1, 77, 16).half()
    for sched, name, steps, strength, t_noise in ((PNDMSchedulerB200(), "PNDMScheduler", 1, 0.8, 1),
                                                  (DPMSolverMultistepSchedulerB200(), "DPMSolverMultistepScheduler", 25,
                                                   0.02, 999)):
        pipe, unet = _pipe(monkeypatch, scheduler=sched)
        out = pipe.interpolate_img2img(text_embeddings=text, init_latents=lat, generator_a=None, generator_b=None,
                                       interpolate_alpha=0.0, strength_a=strength, strength_b=strength,
                                       num_inference_steps=steps, guidance_scale=7.0, uncond_embeddings=uncond,
                                       noise=noise, output_type="latent")
        a = float(sched.alphas_cumprod[t_noise])
        assert out["n_unet_evals"] == 0 and not unet.inputs, name
        assert torch.equal(out["latents_unscaled"], (a ** 0.5 * lat.float() + (1 - a) ** 0.5 * noise.float()).half())
        out = pipe.img2img("", None, strength=strength, num_inference_steps=steps, seed=9, scheduler=name,
                           output_type="latent", text_embeddings=text, uncond_embeddings=uncond, moments=(mean, logvar))
        assert out["n_unet_evals"] == 0 and not unet.inputs and out["t_start"] == steps, name
        for i in range(2):
            post = torch.randn((1, 4, 8, 8), generator=torch.Generator().manual_seed(9))
            std = torch.exp(0.5 * torch.clamp(logvar[i:i + 1], -30.0, 20.0))
            clean = VAE_SCALE * (mean[i:i + 1].float() + std.float() * post).half()
            assert torch.equal(out["latents_unscaled"][i:i + 1], clean), name


def test_mismatched_uncond_embeddings_rejected_before_the_unet(monkeypatch):
    """2 uncond rows for 3 clips would concatenate into a 5-row context; txt2img, img2img and interpolate_img2img raise
    ValueError before the UNet runs"""
    pipe, unet = _pipe(monkeypatch)
    torch.manual_seed(7)
    text, uncond = torch.randn(3, 77, 16).half(), torch.randn(2, 77, 16).half()
    lat, logvar = torch.randn(3, 4, 8, 8).half(), torch.zeros(3, 4, 8, 8).half()
    runs = [
        lambda: pipe.txt2img("", num_clips=3, num_inference_steps=5, width=64, height=64, output_type="latent",
                             text_embeddings=text, uncond_embeddings=uncond),
        lambda: pipe.img2img("", None, num_inference_steps=5, output_type="latent", text_embeddings=text,
                             uncond_embeddings=uncond, moments=(lat, logvar)),
        lambda: pipe.interpolate_img2img(text_embeddings=text, init_latents=lat, generator_a=None, generator_b=None,
                                         interpolate_alpha=0.0, num_inference_steps=5, uncond_embeddings=uncond,
                                         noise=torch.randn(3, 4, 8, 8).half(), output_type="latent"),
    ]
    for run in runs:
        with pytest.raises(ValueError, match="uncond_embeddings hold 2 rows for 3 clips"):
            run()
        assert not unet.inputs


# ----------------------------------------------------------------------------------------------- CLI
def test_cli_audio_to_audio_command_and_flags():
    """`main` offers audio-to-audio; build_parser() alone still builds exactly the reference's six commands"""
    from riffusion import cli

    sub = next(a for a in cli.build_parser()._actions if a.dest == "command")
    assert set(sub.choices) == {"audio-to-image", "image-to-audio", "sample-clips", "print-exif",
                                "audio-to-images-batch", "sample-clips-batch"}
    parser = cli.build_parser(cli.COMMANDS + cli.EXTRA_COMMANDS + cli.TRACK_COMMANDS)
    sub = next(a for a in parser._actions if a.dest == "command")
    assert "audio-to-audio" in sub.choices and "text-to-audio" in sub.choices
    flags = {o for act in sub.choices["audio-to-audio"]._actions for o in act.option_strings}
    assert {"--audio", "--output", "--prompt", "--image-dir", "--negative-prompt", "--seed", "--denoising",
            "--num-inference-steps", "--guidance", "--scheduler", "--start-time-s", "--duration-s", "--clip-duration-s",
            "--overlap-duration-s", "--prompt-b", "--seed-b", "--denoising-b", "--max-batch", "--use-20k",
            "--checkpoint", "--device"} <= flags
    ns = parser.parse_args(["audio-to-audio", "--audio", "in.wav", "--output", "o.wav", "--prompt", "jazz"])
    assert (ns.seed, ns.denoising, ns.num_inference_steps, ns.guidance, ns.scheduler) == \
        (42, 0.55, 25, 7.0, "DPMSolverMultistepScheduler")
    assert (ns.start_time_s, ns.duration_s, ns.clip_duration_s, ns.overlap_duration_s, ns.use_20k, ns.max_batch) == \
        (0.0, 20.0, 5.0, 0.2, False, 32)


def test_cli_audio_to_audio_writes_files(monkeypatch, tmp_path):
    """through `main` with the checkpoint loader replaced by a recorder: the arguments reach audio_to_audio, the stitched
    track is written, and --image-dir gets each clip's source and riffed PNG with the params in the EXIF"""
    from riffusion import cli
    from riffusion.riffusion_pipeline import RiffusionPipeline
    from riffusion.spectrogram_params import SpectrogramParams
    from riffusion.util.audio_util import AudioSegment

    calls = {}

    class FakePipe:
        def audio_to_audio(self, track, prompt, **kw):
            calls.update(kw, prompt=prompt, track=track)
            seg = AudioSegment(np.zeros((44100 * 2, 2), np.int16), 44100)
            img = torch.full((2, 512, 501, 3), 7, dtype=torch.uint8)
            return dict(segment=seg, source_images=img, images=img + 1, clip_start_times=np.array([0.0, 4.8]))

    def load(cls, checkpoint, device):
        calls.update(checkpoint=checkpoint, device=device)
        return FakePipe()

    monkeypatch.setattr(RiffusionPipeline, "load_checkpoint", classmethod(load))
    _track(12.0).export(str(tmp_path / "in.wav"), format="wav")
    cli.main(["audio-to-audio", "--audio", str(tmp_path / "in.wav"), "--output", str(tmp_path / "out.wav"), "--prompt",
              "jazz", "--use-20k", "--image-dir", str(tmp_path / "img"), "--prompt-b", "rock", "--seed-b", "7",
              "--denoising", "0.4", "--checkpoint", "ckpt"])
    want = SpectrogramParams(min_frequency=10, max_frequency=20000, stereo=True)
    assert calls["prompt"] == "jazz" and calls["params"] == want and calls["prompt_b"] == "rock"
    assert (calls["seed"], calls["seed_b"], calls["denoising"], calls["denoising_b"], calls["negative_prompt"]) == \
        (42, 7, 0.4, None, None)
    assert (calls["num_inference_steps"], calls["guidance_scale"], calls["max_batch"], calls["checkpoint"]) == \
        (25, 7.0, 32, "ckpt")
    assert abs(calls["track"].duration_seconds - 12.0) < 1e-9
    assert AudioSegment.from_file(str(tmp_path / "out.wav")).channels == 2
    for i in range(2):
        for kind, v in (("source", 7), ("riffed", 8)):
            img = Image.open(tmp_path / "img" / f"clip_{i}_{kind}.png")
            assert img.size == (501, 512) and np.asarray(img)[0, 0, 0] == v
            assert SpectrogramParams.from_exif(img.getexif()) == want


# ----------------------------------------------------------------------------------------------- bench
def test_bench_script_accounting():
    spec = importlib.util.spec_from_file_location("bench_audio_to_audio", ROOT / "tools" / "bench_audio_to_audio.py")
    mod = importlib.util.module_from_spec(spec)
    sys.modules["bench_audio_to_audio"] = mod
    spec.loader.exec_module(mod)
    assert mod.output_seconds(4, 5.0, 0.2) == pytest.approx(19.4)
    assert mod.output_seconds(12, 5.0, 0.2) == pytest.approx(57.8)
