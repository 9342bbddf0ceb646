"""Magic Mix on the host: the (t_max, t_min) rule and evaluation counts of both schedulers, the control flow of
RiffusionPipeline.magic_mix with the device steps replaced by their torch definitions (layout-phase UNet inputs, the
sample the scheduler steps, the noise and posterior draws), its reduction to img2img, the audio_to_audio rejections and
the `audio-to-audio` flags.  The algorithm restates diffusers' community pipeline from memory (unpinned)."""
import importlib.util
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]
DPM, PNDM = "DPMSolverMultistepScheduler", "PNDMScheduler"


def _fake_magic_mix(x, enc, noise, a, b, mix):
    """torch definition of rf_magic_mix_f16"""
    assert noise.dtype == torch.float32
    return (mix * x.float() + (1 - mix) * (a * enc.float() + b * noise)).half()


def _mm_pipe(monkeypatch):
    """the recording-UNet pipeline of test_audio_to_audio_cpu, plus the torch magic_mix and a scheduler double that
    records the sample every step is given and the sample it returns"""
    from test_audio_to_audio_cpu import _pipe

    from riffusion import riffusion_pipeline as rp
    from riffusion import tc_ops
    from riffusion.scheduler_b200 import make_scheduler

    calls = []
    monkeypatch.setattr(tc_ops, "magic_mix", lambda *a: calls.append(a) or _fake_magic_mix(*a))
    scheds = []

    class StepRecorder:
        def __init__(self, inner):
            self.inner, self.samples, self.outs = inner, [], []

        def __getattr__(self, name):
            return getattr(self.inner, name)

        def step_cfg(self, eps_pair, guidance, t, sample):
            self.samples.append(sample.clone())
            out = self.inner.step_cfg(eps_pair, guidance, t, sample)
            self.outs.append(out.clone())
            return out

    def make(name):
        scheds.append(StepRecorder(make_scheduler(name)))
        return scheds[-1]

    monkeypatch.setattr(rp, "make_scheduler", make)
    pipe, unet = _pipe(monkeypatch)
    return pipe, unet, scheds, calls


def _inputs(n=3, seed=3):
    torch.manual_seed(seed)
    mean = torch.randn(n, 4, 8, 8).half()
    logvar = (torch.randn(n, 4, 8, 8) * 0.5 - 2).half()
    text, uncond = torch.randn(1, 77, 16).half(), torch.randn(1, 77, 16).half()
    return mean, logvar, text, uncond


def _enc(mean, logvar, seed):
    """clip i's posterior sample: its own generator seeded with `seed`, fp32 draw (here a CPU generator: the pipeline
    runs on the CPU)"""
    from riffusion.riffusion_pipeline import VAE_SCALE

    rows = []
    for i in range(mean.shape[0]):
        post = torch.randn((1, 4, 8, 8), generator=torch.Generator().manual_seed(seed))
        std = torch.exp(0.5 * torch.clamp(logvar[i:i + 1], -30.0, 20.0))
        rows.append(VAE_SCALE * (mean[i:i + 1].float() + std.float() * post).half())
    return torch.cat(rows)


# ----------------------------------------------------------------------------------------------- M1
@pytest.mark.parametrize("n,kmin,kmax,t_max,t_min", [(25, 0.3, 0.5, 13, 18), (10, 0.2, 0.8, 2, 8), (20, 0.3, 0.5, 10, 14),
                                                     (7, 0.3, 0.5, 4, 5), (25, 0.6, 0.5, 13, 10), (4, 0.0, 1.0, 0, 4),
                                                     (3, 0.1, 0.34, 2, 3)])
def test_range_eval_counts_and_timesteps(monkeypatch, n, kmin, kmax, t_max, t_min):
    """t_max = n - int(kmax n), t_min = n - int(kmin n); the UNet sees T[t_max:], len(T) - t_max evaluations: n - t_max
    for DPM-Solver++ and one more for PNDM, whose table repeats a timestep"""
    from riffusion.riffusion_pipeline import RiffusionPipeline

    assert RiffusionPipeline.magic_mix_range(n, kmin, kmax) == (t_max, t_min)
    pipe, unet, scheds, _ = _mm_pipe(monkeypatch)
    mean, logvar, text, uncond = _inputs(2)
    for name, extra in ((DPM, 0), (PNDM, 1)):
        unet.inputs.clear()
        unet.timesteps.clear()
        out = pipe.magic_mix("", None, kmin=kmin, kmax=kmax, num_inference_steps=n, scheduler=name, output_type="latent",
                             text_embeddings=text, uncond_embeddings=uncond, moments=(mean, logvar))
        T_ = scheds[-1].timesteps
        assert len(T_) == n + extra
        assert out["n_unet_evals"] == len(unet.inputs) == n + extra - t_max, name
        assert (out["t_max"], out["t_min"]) == (t_max, t_min)
        assert unet.timesteps == [int(t) for t in T_[t_max:]], name
        assert out["images"] is None and out["latents_unscaled"].shape == (2, 4, 8, 8)


def test_n25_defaults_example(monkeypatch):
    """25 steps with the app's kmin 0.3 / kmax 0.5: t_max 13, t_min 18, 12 evaluations for DPM-Solver++ and 13 for PNDM,
    and the steps i = 14..17 are mixed"""
    pipe, unet, scheds, calls = _mm_pipe(monkeypatch)
    mean, logvar, text, uncond = _inputs(1)
    for name, evals in ((DPM, 12), (PNDM, 13)):
        calls.clear()
        out = pipe.magic_mix("", None, scheduler=name, output_type="latent", text_embeddings=text,
                             uncond_embeddings=uncond, moments=(mean, logvar))
        assert (out["t_max"], out["t_min"], out["n_unet_evals"]) == (13, 18, evals)
        T_ = scheds[-1].timesteps
        # the first call is the noising at T[13] (mix 0); then one blend per layout step, at T[14..17]
        assert [c[5] for c in calls] == [0.0, 0.5, 0.5, 0.5, 0.5]
        ab = scheds[-1].alphas_cumprod
        assert [c[3] for c in calls] == [float(ab[int(T_[i])]) ** 0.5 for i in (13, 14, 15, 16, 17)]


@pytest.mark.parametrize("n,kmax", [(25, 0.03), (3, 0.3), (10, 0.05), (1, 0.99)])
def test_kmax_below_one_step_rejected(monkeypatch, n, kmax):
    """int(kmax * n) == 0 would start at T[n], past the end of the table: ValueError before the UNet runs"""
    pipe, unet, _, _ = _mm_pipe(monkeypatch)
    mean, logvar, text, uncond = _inputs(1)
    assert int(kmax * n) == 0
    for name in (DPM, PNDM):
        with pytest.raises(ValueError, match="kmax"):
            pipe.magic_mix("", None, kmax=kmax, kmin=0.0, num_inference_steps=n, scheduler=name, output_type="latent",
                           text_embeddings=text, uncond_embeddings=uncond, moments=(mean, logvar))
    with pytest.raises(ValueError, match="kmax"):
        pipe.magic_mix("", None, kmax=1.2, output_type="latent", text_embeddings=text, uncond_embeddings=uncond,
                       moments=(mean, logvar))
    assert not unet.inputs


# ----------------------------------------------------------------------------------------------- M2
@pytest.mark.parametrize("name", [DPM, PNDM])
@pytest.mark.parametrize("n,kmin,kmax,mix", [(25, 0.3, 0.5, 0.5), (10, 0.2, 0.8, 0.3)])
def test_layout_and_content_phase_inputs(monkeypatch, name, n, kmin, kmax, mix):
    """x_0 = add_noise(enc, noise, T[t_max]); the scheduler is stepped with x (never u); each layout-phase UNet input is
    mix x + (1 - mix) add_noise(enc, noise, T[i]) of the previous step's output, content-phase inputs are x itself"""
    pipe, unet, scheds, _ = _mm_pipe(monkeypatch)
    mean, logvar, text, uncond = _inputs(3, seed=n)
    out = pipe.magic_mix("", None, kmin=kmin, kmax=kmax, mix_factor=mix, num_inference_steps=n, seed=5, scheduler=name,
                         output_type="latent", text_embeddings=text, uncond_embeddings=uncond, moments=(mean, logvar))
    s = scheds[-1]
    T_ = [int(t) for t in s.timesteps]
    t_max, t_min = out["t_max"], out["t_min"]
    enc = _enc(mean, logvar, 5)
    noise = torch.randn((1, 4, 8, 8), generator=torch.Generator().manual_seed(5))

    def noised(t):
        a = float(s.alphas_cumprod[t])
        return a ** 0.5 * enc.float() + (1 - a) ** 0.5 * noise

    x = noised(T_[t_max]).half()
    assert len(s.samples) == len(unet.inputs) == len(T_) - t_max
    for j, i in enumerate(range(t_max, len(T_))):
        assert torch.equal(s.samples[j], x), (name, i)                                 # the step gets x
        if t_max < i < t_min:
            want = (mix * x.float() + (1 - mix) * noised(T_[i])).half()
            assert not torch.equal(want, x)
        else:
            want = x
        assert torch.equal(unet.inputs[j], torch.cat([want, want])), (name, i)
        x = s.outs[j]
    assert torch.equal(out["latents_unscaled"], x)


def test_noise_and_posterior_draws(monkeypatch):
    """the noise is the fp32 CPU draw torch.randn((1, 4, h, w)) after manual_seed(seed), the same for every clip; each
    clip's posterior sample comes from its own generator seeded with `seed`; an injected (1 or B)-row fp32 noise replaces
    the draw"""
    pipe, unet, _, calls = _mm_pipe(monkeypatch)
    mean, logvar, text, uncond = _inputs(3)
    kw = dict(num_inference_steps=10, seed=17, output_type="latent", text_embeddings=text, uncond_embeddings=uncond,
              moments=(mean, logvar))
    out = pipe.magic_mix("", None, **kw)
    draw = torch.randn((1, 4, 8, 8), generator=torch.Generator().manual_seed(17))
    x, enc, noise, a, b, mix = calls[0]
    assert mix == 0.0 and noise.dtype == torch.float32 and noise.shape == (3, 4, 8, 8)
    for i in range(3):
        assert torch.equal(noise[i:i + 1], draw)
    assert torch.equal(enc, _enc(mean, logvar, 17)) and torch.equal(x, enc)
    assert not torch.equal(enc[0], enc[1])                                             # per-clip moments
    assert all(c[1] is enc and c[2] is noise for c in calls)
    calls.clear()
    again = pipe.magic_mix("", None, noise=draw, **kw)
    assert torch.equal(again["latents_unscaled"], out["latents_unscaled"])
    calls.clear()
    rows = torch.cat([draw, 2 * draw, draw])
    three = pipe.magic_mix("", None, noise=rows, **kw)
    assert torch.equal(calls[0][2], rows)
    assert torch.equal(three["latents_unscaled"][0], out["latents_unscaled"][0])
    assert not torch.equal(three["latents_unscaled"][1], out["latents_unscaled"][1])
    with pytest.raises(ValueError, match="noise must be"):
        pipe.magic_mix("", None, noise=torch.zeros(2, 4, 8, 8), **kw)


def test_uncond_is_the_empty_prompt(monkeypatch):
    """no negative prompt: the unconditional half of the context is embed_text("")"""
    pipe, unet, _, _ = _mm_pipe(monkeypatch)
    mean, logvar, text, _ = _inputs(2)
    seen = []
    empty = torch.full((1, 77, 16), 0.25).half()
    monkeypatch.setattr(type(pipe), "embed_text", lambda self, p: seen.append(p) or empty)
    pipe.magic_mix("", None, num_inference_steps=10, output_type="latent", text_embeddings=text, moments=(mean, logvar))
    assert seen == [""]


# ----------------------------------------------------------------------------------------------- M3
@pytest.mark.parametrize("name", [DPM, PNDM])
@pytest.mark.parametrize("kmin,mix", [(0.3, 1.0), (0.5, 0.5), (0.7, 0.5)])
def test_reduces_to_img2img(monkeypatch, name, kmin, mix):
    """mix_factor 1, or kmin >= kmax (no layout phase): UNet inputs and outputs equal img2img(strength=kmax) on the same
    moments and (fp16-representable) noise"""
    pipe, unet, _, _ = _mm_pipe(monkeypatch)
    mean, logvar, text, uncond = _inputs(2, seed=11)
    noise = torch.randn((1, 4, 8, 8), generator=torch.Generator().manual_seed(4)).half()
    kw = dict(num_inference_steps=25, seed=8, scheduler=name, output_type="latent", text_embeddings=text,
              uncond_embeddings=uncond, moments=(mean, logvar))
    mm = pipe.magic_mix("", None, kmin=kmin, kmax=0.5, mix_factor=mix, noise=noise.float(), **kw)
    mm_inputs = list(unet.inputs)
    unet.inputs.clear()
    ref = pipe.img2img("", None, strength=0.5, noise=noise.expand(2, -1, -1, -1), **kw)
    assert mm["n_unet_evals"] == ref["n_unet_evals"] and mm["t_max"] == ref["t_start"]
    assert len(mm_inputs) == len(unet.inputs)
    for got, want in zip(mm_inputs, unet.inputs):
        assert torch.equal(got, want)
    assert torch.equal(mm["latents_unscaled"], ref["latents_unscaled"])


# ----------------------------------------------------------------------------------------------- M4
def _track(seconds):
    from riffusion.util.audio_util import AudioSegment

    rng = np.random.default_rng(0)
    return AudioSegment(rng.integers(-8000, 8000, size=(int(seconds * 44100), 1)).astype(np.int16), 44100)


def test_audio_to_audio_rejections():
    """magic_mix with prompt_b or a negative prompt (the app asserts both), or with kmax below one step, raises
    ValueError before any device work"""
    from riffusion.riffusion_pipeline import RiffusionPipeline

    pipe = RiffusionPipeline(vae=None, unet=None, device="cpu")
    with pytest.raises(ValueError, match="prompt_b"):
        pipe.audio_to_audio(_track(12.0), "jazz", magic_mix=True, prompt_b="rock")
    with pytest.raises(ValueError, match="negative prompt"):
        pipe.audio_to_audio(_track(12.0), "jazz", magic_mix=True, negative_prompt="noise")
    with pytest.raises(ValueError, match="kmax"):
        pipe.audio_to_audio(_track(12.0), "jazz", magic_mix=True, kmax=0.01)


def test_cli_magic_mix_flags(monkeypatch, tmp_path):
    """--magic-mix, --kmin, --kmax and --mix-factor come from audio_to_audio's signature and reach the pipeline; without
    them the img2img mode runs"""
    from riffusion import cli
    from riffusion.riffusion_pipeline import RiffusionPipeline
    from riffusion.util.audio_util import AudioSegment

    parser = cli.build_parser(cli.COMMANDS + cli.EXTRA_COMMANDS + cli.TRACK_COMMANDS)
    ns = parser.parse_args(["audio-to-audio", "--audio", "in.wav", "--output", "o.wav", "--prompt", "jazz"])
    assert (ns.magic_mix, ns.kmin, ns.kmax, ns.mix_factor) == (False, 0.3, 0.5, 0.5)
    calls = []

    class FakePipe:
        def audio_to_audio(self, track, prompt, **kw):
            calls.append(kw)
            img = torch.zeros((2, 512, 501, 3), dtype=torch.uint8)
            return dict(segment=AudioSegment(np.zeros((44100, 1), np.int16), 44100), source_images=img, images=img,
                        clip_start_times=np.array([0.0, 4.8]))

    monkeypatch.setattr(RiffusionPipeline, "load_checkpoint", classmethod(lambda cls, **kw: FakePipe()))
    _track(12.0).export(str(tmp_path / "in.wav"), format="wav")
    base = ["audio-to-audio", "--audio", str(tmp_path / "in.wav"), "--output", str(tmp_path / "out.wav"), "--prompt",
            "jazz"]
    cli.main(base + ["--magic-mix", "--kmin", "0.2", "--kmax", "0.7", "--mix-factor", "0.4", "--scheduler", PNDM])
    cli.main(base)
    assert (calls[0]["magic_mix"], calls[0]["kmin"], calls[0]["kmax"], calls[0]["mix_factor"]) == (True, 0.2, 0.7, 0.4)
    assert calls[0]["scheduler"] == PNDM and calls[0]["negative_prompt"] is None and calls[0]["prompt_b"] is None
    assert (calls[1]["magic_mix"], calls[1]["kmin"], calls[1]["kmax"], calls[1]["mix_factor"]) == (False, 0.3, 0.5, 0.5)


def test_bench_magic_mix_evals():
    spec = importlib.util.spec_from_file_location("bench_audio_to_audio", ROOT / "tools" / "bench_audio_to_audio.py")
    mod = importlib.util.module_from_spec(spec)
    sys.modules["bench_audio_to_audio"] = mod
    spec.loader.exec_module(mod)
    assert mod.magic_mix_evals(25, 0.5, DPM) == 12 and mod.magic_mix_evals(25, 0.5, PNDM) == 13
    assert mod.magic_mix_evals(10, 0.8, DPM) == 8 and mod.magic_mix_evals(10, 0.8, PNDM) == 9
