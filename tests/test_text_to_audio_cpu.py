"""Text-to-audio on the host: the DPM-Solver++ scheduler's bookkeeping against the oracle restatement, an independent
pin of its convergence order, the control flow of RiffusionPipeline.txt2img / text_to_audio with the device steps
replaced by their torch definitions, the `text-to-audio` command's flags and the benchmark script's accounting."""
import importlib.util
import sys
import types
from pathlib import Path

import pytest
import torch

from txt2img_oracle import DPMSolverMultistepOracle, txt2img_loop

ROOT = Path(__file__).resolve().parents[1]


def _fake_dpm_step(eps_pair, guidance, sample, m1, coefs):
    """torch definition of rf_cfg_dpmpp_step_f16, in the dtype of the inputs"""
    alpha_s0, sigma_s0, c_x, c_0, c_1 = coefs
    n = sample.shape[0]
    eu, et = eps_pair[:n], eps_pair[n:]
    eps = eu + guidance * (et - eu)
    x0 = (sample - sigma_s0 * eps) / alpha_s0
    prev = c_x * sample + c_0 * x0
    if m1 is not None:
        prev = prev + c_1 * (x0 - m1)
    return x0, prev


def _fake_pndm_step(eps_pair, guidance, hist, coef, sample, ca, cb, want_eps=True):
    n = sample.shape[0]
    eu, et = eps_pair[:n].float(), eps_pair[n:].float()
    eps = eu + guidance * (et - eu)
    e = coef[0] * eps
    for c, h in zip(coef[1:], hist):
        e = e + c * h.float()
    return (eps.to(sample.dtype) if want_eps else None), (ca * sample.float() - cb * e).to(sample.dtype)


# ----------------------------------------------------------------------------------------------- C1
def test_dpm_tables_match_oracle():
    from riffusion.scheduler_b200 import DPMSolverMultistepSchedulerB200

    ours, ref = DPMSolverMultistepSchedulerB200(), DPMSolverMultistepOracle(dtype=torch.float64)
    for n in (5, 10, 14, 15, 30, 50):
        ours.set_timesteps(n)
        ref.set_timesteps(n)
        assert ours.timesteps.tolist() == ref.timesteps.tolist()
        assert ours.timesteps[0] == 999 and len(ours.timesteps) == n and ours.timesteps[-1] > 0
    ours.set_timesteps(30)
    assert ours.timesteps.tolist()[:3] == [999, 966, 932] and ours.timesteps.tolist()[-1] == 33
    assert torch.equal(ours.alphas_cumprod, ref.alphas_cumprod)
    assert torch.allclose(torch.from_numpy(ours.alpha_t), ref.alpha_t, rtol=1e-14, atol=0)
    assert torch.allclose(torch.from_numpy(ours.sigma_t), ref.sigma_t, rtol=1e-14, atol=0)
    assert torch.allclose(torch.from_numpy(ours.lambda_t), ref.lambda_t, rtol=1e-13, atol=1e-13)
    assert ours.init_noise_sigma == 1.0 and torch.equal(ours.scale_model_input(ref.alpha_t), ref.alpha_t)


@pytest.mark.parametrize("n", [5, 10, 14, 15, 30])
def test_dpm_scheduler_bookkeeping_matches_oracle(monkeypatch, n):
    """host side of DPMSolverMultistepSchedulerB200 (step index, previous timestep, first / last step order, history,
    fp64 coefficients) step by step against the oracle scheduler, with the fused device kernel replaced by its torch
    definition; 14 and 15 steps sit on both sides of lower_order_final's `< 15` rule"""
    from riffusion import tc_ops
    from riffusion.scheduler_b200 import DPMSolverMultistepSchedulerB200

    monkeypatch.setattr(tc_ops, "cfg_dpmpp_step", _fake_dpm_step)
    ours, ref = DPMSolverMultistepSchedulerB200(), DPMSolverMultistepOracle(dtype=torch.float64)
    ours.set_timesteps(n)
    ref.set_timesteps(n)
    torch.manual_seed(n)
    x_o = x_r = torch.randn(2, 4, 8, 8, dtype=torch.float64)
    g = 7.0
    orders = []
    for t in ref.timesteps.tolist():
        orders.append(ours.plan(t)[0])
        pair = torch.randn(4, 4, 8, 8, dtype=torch.float64)
        x_r = ref.step(pair[:2] + g * (pair[2:] - pair[:2]), t, x_r)
        x_o = ours.step_cfg(pair, g, t, x_o)
        assert torch.allclose(x_o, x_r, rtol=1e-10, atol=1e-10), t
    assert orders[0] == 1 and all(o == 2 for o in orders[1:-1])
    assert orders[-1] == (1 if n < 15 else 2)
    # the diffusers-style step with an already guided model output gives the same result
    ours.set_timesteps(n)
    ref.set_timesteps(n)
    x_o = x_r = torch.randn(1, 4, 8, 8, dtype=torch.float64)
    for t in ref.timesteps.tolist()[:4]:
        eps = torch.randn(1, 4, 8, 8, dtype=torch.float64)
        x_r = ref.step(eps, t, x_r)
        x_o = ours.step(eps, t, x_o).prev_sample
    assert torch.allclose(x_o, x_r, rtol=1e-10, atol=1e-10)


# ----------------------------------------------------------------------------------------------- C3
def _gaussian_run(scheduler_step, set_timesteps, timesteps, a, sg, s2):
    """probability-flow ODE of Gaussian data x0 ~ N(0, s2 I) with the exact noise prediction
    eps*(x, t) = sigma_t x / (alpha_t^2 s2 + sigma_t^2); returns (final state, exact final state)"""
    set_timesteps()
    v = lambda t: a[t] ** 2 * s2 + sg[t] ** 2                                  # noqa: E731
    x = torch.linspace(-2.0, 2.0, 9, dtype=torch.float64)
    x_T = x.clone()
    for t in timesteps():
        x = scheduler_step(sg[t] * x / v(t), t, x)
    return x, x_T * torch.sqrt(v(0) / v(999))


@pytest.mark.parametrize("order,lo,hi", [(2, 3.0, 5.0), (1, 1.5, 2.5)])
def test_dpm_convergence_order_on_gaussian_data(monkeypatch, order, lo, hi):
    """Independent pin of the scheduler math (diffusers is not installable).  For Gaussian data the probability-flow ODE
    has the closed form x_t = x_T sqrt(v_t / v_T), v_t = alpha_t^2 s^2 + sigma_t^2, exact on the discrete ab table.
    The fp64 oracle runs from t = 999 to t = 0 on its own timestep tables; the final-state error must fall by ~4 per
    doubling of the step count for solver_order=2 and by ~2 for solver_order=1.  The step counts are 128, 256, 512:
    the timestep table is uniform in t, so the last steps before t = 0 span wide lambda intervals that shrink only
    logarithmically with n, and at 32 / 64 steps the second-order ratio is still 2.9-3.0 (measured).  The B200 class's
    host coefficients, with the device step replaced by its torch definition, reproduce the oracle's run."""
    from riffusion import tc_ops
    from riffusion.scheduler_b200 import DPMSolverMultistepSchedulerB200

    monkeypatch.setattr(tc_ops, "cfg_dpmpp_step", _fake_dpm_step)
    s2 = 1.0
    errs = []
    for n in (128, 256, 512):
        ref = DPMSolverMultistepOracle(solver_order=order, dtype=torch.float64)
        x, exact = _gaussian_run(ref.step, lambda: ref.set_timesteps(n), lambda: ref.timesteps.tolist(), ref.alpha_t,
                                 ref.sigma_t, s2)
        errs.append(float((x - exact).norm() / exact.norm()))
        ours = DPMSolverMultistepSchedulerB200(solver_order=order)

        def step(eps, t, x_):
            return ours.step(eps, t, x_).prev_sample

        x_b, _ = _gaussian_run(step, lambda: ours.set_timesteps(n), lambda: ours.timesteps.tolist(), ref.alpha_t,
                               ref.sigma_t, s2)
        assert torch.allclose(x_b, x, rtol=1e-11, atol=1e-12), n
    ratios = [errs[0] / errs[1], errs[1] / errs[2]]
    print(f"solver_order={order}: errors {errs}, ratios per doubling {ratios}")
    assert all(lo <= r <= hi for r in ratios), (errs, ratios)


# ----------------------------------------------------------------------------------------------- C2
class _RecordingUNet:
    def __init__(self):
        self.inputs = []

    def __call__(self, x, t, encoder_hidden_states=None, **kw):
        self.inputs.append(x.clone())
        out = 0.3 * torch.tanh(x.float()) + 0.002 * (t / 1000.0) + \
            0.05 * encoder_hidden_states.float().mean(dim=(1, 2))[:, None, None, None]
        return types.SimpleNamespace(sample=out.to(torch.float16))


def _pipe(monkeypatch):
    from riffusion import tc_ops
    from riffusion.riffusion_pipeline import RiffusionPipeline

    def dpm(eps_pair, guidance, sample, m1, coefs):
        x0, prev = _fake_dpm_step(eps_pair.float(), guidance, sample.float(), None if m1 is None else m1.float(), coefs)
        return x0.half(), prev.half()

    monkeypatch.setattr(tc_ops, "cfg_dpmpp_step", dpm)
    monkeypatch.setattr(tc_ops, "cfg_pndm_step", _fake_pndm_step)
    unet = _RecordingUNet()
    pipe = RiffusionPipeline(vae=None, unet=unet, device="cpu")
    pipe.use_cuda_graph = False
    return pipe, unet


def test_txt2img_control_flow(monkeypatch):
    """evaluation counts, per-clip seeds, the oracle loop, argument checks"""
    from oracle import unet_oracle as uo

    pipe, unet = _pipe(monkeypatch)
    torch.manual_seed(4)
    text, uncond = torch.randn(1, 77, 16).half(), torch.randn(1, 77, 16).half()
    for sched, steps, n_want in (("DPMSolverMultistepScheduler", 12, 12), ("DPMSolverMultistepScheduler", 30, 30),
                                 ("PNDMScheduler", 10, 11)):
        unet.inputs.clear()
        out = pipe.txt2img("", seed=7, num_clips=3, num_inference_steps=steps, width=128, height=64, scheduler=sched,
                           output_type="latent", text_embeddings=text, uncond_embeddings=uncond)
        assert out["n_unet_evals"] == n_want == len(unet.inputs)
        first = unet.inputs[0]
        assert first.shape == (6, 4, 8, 16)
        for i in range(3):                                 # clip i draws from a generator seeded with seed + i
            want = torch.randn((1, 4, 8, 16), generator=torch.Generator().manual_seed(7 + i), dtype=torch.float16)
            assert torch.equal(first[i:i + 1], want) and torch.equal(first[3 + i:4 + i], want)
        lat0 = first[:3]
        sch = DPMSolverMultistepOracle() if sched.startswith("DPM") else uo.PNDMSchedulerOracle()
        ref, n_ref = txt2img_loop(lambda x, t, c: unet.__call__(x.half(), t, c.half()).sample.float(), sch,
                                  text.float().expand(3, -1, -1), uncond.float().expand(3, -1, -1), lat0.float(), steps, 7.0)
        assert n_ref == n_want
        err = float((out["latents_unscaled"].float() - ref).norm() / ref.norm())
        assert err < 2e-2, (sched, steps, err)
        assert torch.equal(out["latents"], (1.0 / 0.18215) * out["latents_unscaled"])
    assert pipe.scheduler.timesteps.tolist()[:2] == [981, 961]            # riffuse's PNDM instance is untouched
    with pytest.raises(ValueError, match="multiples of 64"):
        pipe.txt2img("", width=500, text_embeddings=text, uncond_embeddings=uncond)
    with pytest.raises(ValueError, match="DPMSolverMultistepScheduler, PNDMScheduler"):
        pipe.txt2img("", scheduler="EulerDiscreteScheduler", text_embeddings=text, uncond_embeddings=uncond)
    with pytest.raises(ValueError, match="num_frequencies"):
        pipe.text_to_audio("", height=256, text_embeddings=text, uncond_embeddings=uncond)


def test_txt2img_injected_latents_and_prompts(monkeypatch):
    """injected latents are used as they are; the prompt and the negative prompt go through plain embed_text"""
    pipe, unet = _pipe(monkeypatch)
    seen = []
    emb = {"jazz": torch.full((1, 77, 16), 0.5).half(), "": torch.zeros(1, 77, 16).half(), "noise": torch.ones(1, 77, 16).half()}
    pipe.embed_text = lambda text: seen.append(text) or emb[text]
    lat = torch.randn(2, 4, 8, 8).half()
    pipe.txt2img("jazz", num_clips=2, num_inference_steps=5, width=64, height=64, output_type="latent", latents=lat)
    assert seen == ["jazz", ""] and torch.equal(unet.inputs[0][:2], lat)
    seen.clear()
    pipe.txt2img("jazz", negative_prompt="noise", num_clips=2, num_inference_steps=5, width=64, height=64,
                 output_type="latent", latents=lat)
    assert seen == ["jazz", "noise"]
    with pytest.raises(ValueError, match="latents must be"):
        pipe.txt2img("jazz", num_clips=3, num_inference_steps=5, width=64, height=64, output_type="latent", latents=lat)


# ----------------------------------------------------------------------------------------------- C4
def test_cli_text_to_audio_command_and_flags(monkeypatch):
    """`main` offers text-to-audio next to the reference's six commands (build_parser() alone stays the reference's
    surface); its flags, defaults, and the arguments it hands to the pipeline"""
    from riffusion import cli

    assert [f.__name__ for f in cli.EXTRA_COMMANDS] == ["text_to_audio"]
    parser = cli.build_parser(cli.COMMANDS + cli.EXTRA_COMMANDS)
    sub = next(a for a in parser._actions if a.dest == "command")
    assert set(sub.choices) == {"audio-to-image", "image-to-audio", "sample-clips", "print-exif",
                                "audio-to-images-batch", "sample-clips-batch", "text-to-audio"}
    t2a = {o for act in sub.choices["text-to-audio"]._actions for o in act.option_strings}
    assert {"--prompt", "--audio", "--image", "--negative-prompt", "--seed", "--num-clips", "--num-inference-steps",
            "--guidance", "--width", "--scheduler", "--use-20k", "--checkpoint", "--device"} <= t2a
    ns = parser.parse_args(["text-to-audio", "--prompt", "jazz", "--audio", "o.wav", "--use-20k", "--num-clips", "3",
                            "--guidance", "6.5", "--negative-prompt", "noise"])
    assert (ns.prompt, ns.audio, ns.use_20k, ns.num_clips, ns.guidance, ns.negative_prompt) == ("jazz", "o.wav", True, 3, 6.5, "noise")
    assert (ns.seed, ns.num_inference_steps, ns.width, ns.scheduler, ns.image) == (42, 30, 512, "DPMSolverMultistepScheduler", "")


def test_cli_text_to_audio_writes_files(monkeypatch, tmp_path):
    """`python -m riffusion.cli text-to-audio` through `main`, with the checkpoint loader replaced by a recorder that
    returns host tensors: the arguments reach text_to_audio, clip i is written as out_<seed + i>.wav / .png, and the
    PNG's EXIF holds the 20 kHz stereo params"""
    from PIL import Image

    from riffusion import cli
    from riffusion.riffusion_pipeline import RiffusionPipeline
    from riffusion.spectrogram_params import SpectrogramParams
    from riffusion.util.audio_util import AudioSegment

    calls = {}

    class FakePipe:
        def text_to_audio(self, prompt, **kw):
            calls.update(kw, prompt=prompt)
            n, C, W = kw["num_clips"], 2 if kw["params"].stereo else 1, kw["width"]
            wave = torch.sin(torch.arange(441 * (W - 1), dtype=torch.float32) / 7.0).repeat(n, C, 1)
            return dict(images=torch.full((n, 512, W, 3), 100, dtype=torch.uint8), waveform=wave)

    def load(cls, checkpoint, device):
        calls.update(checkpoint=checkpoint, device=device)
        return FakePipe()

    monkeypatch.setattr(RiffusionPipeline, "load_checkpoint", classmethod(load))
    cli.main(["text-to-audio", "--prompt", "jazz", "--audio", str(tmp_path / "out.wav"), "--image", str(tmp_path / "out.png"),
              "--num-clips", "2", "--seed", "5", "--use-20k", "--width", "256", "--negative-prompt", "noise",
              "--checkpoint", "ckpt", "--device", "cuda:1"])
    want = SpectrogramParams(min_frequency=10, max_frequency=20000, stereo=True)
    assert calls["prompt"] == "jazz" and calls["params"] == want and calls["negative_prompt"] == "noise"
    assert (calls["seed"], calls["num_clips"], calls["width"], calls["guidance_scale"], calls["num_inference_steps"]) == (5, 2, 256, 7.0, 30)
    assert (calls["checkpoint"], calls["device"], calls["scheduler"]) == ("ckpt", "cuda:1", "DPMSolverMultistepScheduler")
    for s in (5, 6):
        seg = AudioSegment.from_file(str(tmp_path / f"out_{s}.wav"))
        assert seg.channels == 2 and seg.frame_rate == 44100 and abs(seg.duration_seconds - 441 * 255 / 44100) < 1e-3
        img = Image.open(tmp_path / f"out_{s}.png")
        assert img.size == (256, 512) and SpectrogramParams.from_exif(img.getexif()) == want


def test_bench_script_accounting():
    spec = importlib.util.spec_from_file_location("bench_text_to_audio", ROOT / "tools" / "bench_text_to_audio.py")
    mod = importlib.util.module_from_spec(spec)
    sys.modules["bench_text_to_audio"] = mod
    spec.loader.exec_module(mod)
    assert mod.n_unet_evals("DPMSolverMultistepScheduler", 30) == 30
    assert mod.n_unet_evals("PNDMScheduler", 30) == 31 and mod.n_unet_evals("PNDMScheduler", 50) == 51
    with pytest.raises(ValueError):
        mod.n_unet_evals("LMSDiscreteScheduler", 30)
    assert mod.tc_tflops(2e12, 1000.0) == pytest.approx(2.0)
    assert mod.audio_samples(768) == 338247 and mod.audio_samples(512) == 225351
