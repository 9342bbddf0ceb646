"""DDIM and Euler ancestral without a GPU: their tables, their steps against independent fp64 restatements, their
convergence on Gaussian data, the pipeline's control flow and draws with the device steps replaced by their torch
definitions, the operand contract of `cfg_euler_a_step`, and the refusals that stay (LMS, plain Euler, Euler ancestral
in Magic Mix, DDIM with eta != 0)."""
import importlib.util
import sys
import types
from pathlib import Path

import numpy as np
import pytest
import torch

from scheduler_oracle import DDIMOracle, EulerAncestralOracle
from test_op_contracts_cpu import recorder  # noqa: F401  (fixture)
from test_text_to_audio_batch_cpu import batch_pipe, _u8  # noqa: F401  (fixture)

ROOT = Path(__file__).resolve().parents[1]
DPM, PNDM, DDIM, EA = "DPMSolverMultistepScheduler", "PNDMScheduler", "DDIMScheduler", "EulerAncestralDiscreteScheduler"


def _fake_euler_a(eps_pair, guidance, guidance_rows, sample, noise, dt, sigma_up):
    """torch definition of rf_cfg_euler_a_step_f16 in fp64, returned in the sample's dtype"""
    d, B = torch.float64, sample.shape[0]
    g = guidance if guidance_rows is None else guidance_rows.to(d).view(-1, *[1] * (sample.dim() - 1))
    eu, et = eps_pair[:B].to(d), eps_pair[B:].to(d)
    prev = sample.to(d) + dt * (eu + g * (et - eu))
    if noise is not None:
        prev = prev + sigma_up * noise.to(d)
    return prev.to(sample.dtype)


def _pndm64(eps_pair, guidance, hist, coef, sample, ca, cb, want_eps=True):
    """torch definition of rf_cfg_pndm_step_f16 in fp64, coefficients unrounded"""
    d, B = torch.float64, sample.shape[0]
    eu, et = eps_pair[:B].to(d), eps_pair[B:].to(d)
    eps = eu + guidance * (et - eu)
    e = coef[0] * eps
    for c, h in zip(coef[1:], hist):
        e = e + c * h.to(d)
    return (eps.to(sample.dtype) if want_eps else None), (ca * sample.to(d) - cb * e).to(sample.dtype)


def _axpby64(x, noise, a, b, mask=None, z=None):
    return (a * x.to(torch.float64) + b * noise.to(torch.float64)).to(x.dtype)


@pytest.fixture
def fake_steps(monkeypatch):
    from test_interpolation_cpu import _fake_rows_step

    from riffusion import scheduler_b200, tc_ops

    monkeypatch.setattr(tc_ops, "cfg_pndm_step", _pndm64)
    monkeypatch.setattr(tc_ops, "axpby", _axpby64)
    monkeypatch.setattr(scheduler_b200, "cfg_pndm_rows_step", _fake_rows_step)
    monkeypatch.setattr(scheduler_b200, "cfg_euler_a_step", _fake_euler_a)


# ----------------------------------------------------------------------------------------------- DDIM
@pytest.mark.parametrize("n", [5, 10, 25, 50])
def test_ddim_timesteps(n):
    from riffusion.scheduler_b200 import DDIMSchedulerB200, make_scheduler

    s = make_scheduler(DDIM)
    assert isinstance(s, DDIMSchedulerB200) and s.config["steps_offset"] == 1 and s.init_noise_sigma == 1.0
    s.set_timesteps(n)
    ratio = 1000 // n
    assert s.timesteps.dtype == torch.int64 and s.timesteps.tolist() == [ratio * k + 1 for k in range(n)][::-1]
    if n == 50:
        assert s.timesteps.tolist()[:3] == [981, 961, 941] and s.timesteps.tolist()[-1] == 1


def test_ddim_step_matches_x0_form(fake_steps):
    """every step of DDIMSchedulerB200 (PNDM's (ca, cb) through the PLMS kernel's torch definition) against the
    oracle's x0-then-direction form, fp64, to 1e-12; the identity checked at 741 -> 721 as well"""
    from riffusion.scheduler_b200 import DDIMSchedulerB200

    ours, ref = DDIMSchedulerB200(), DDIMOracle()
    for n in (10, 50):
        ours.set_timesteps(n)
        ref.set_timesteps(n)
        gen = torch.Generator().manual_seed(n)
        x_o = x_r = torch.randn((2, 4, 3, 5), generator=gen, dtype=torch.float64)
        for t in ref.timesteps.tolist():
            eps = torch.randn((2, 4, 3, 5), generator=gen, dtype=torch.float64)
            x_r = ref.step(eps, t, x_r)
            x_o = ours.step(eps, t, x_o).prev_sample
            assert torch.allclose(x_o, x_r, rtol=1e-12, atol=1e-12), (n, t)
    ours.set_timesteps(50)
    _, cb = ours.coefficients(741, 721)
    assert abs(-cb - -0.08365654740501913) < 1e-12
    coef, hist, override, push, ca, cb2 = ours.plan(741)
    assert (coef, hist, override, push) == ((1.0, 0.0, 0.0, 0.0), [], None, False) and cb2 == cb


def test_ddim_convergence_order_on_gaussian_data(fake_steps):
    """Gaussian data x0 ~ N(0, 1): the probability-flow ODE has the closed form x_t = x_T sqrt(v_t / v_T), v_t = ab_t s^2
    + 1 - ab_t, and DDIM is its first-order solver: the relative final-state error falls ~2x per doubling of n"""
    from riffusion.scheduler_b200 import DDIMSchedulerB200

    ab = DDIMOracle().ab
    v = lambda t: ab[t] + 1 - ab[t]                        # noqa: E731  (s^2 = 1)
    errs = []
    for n in (50, 100, 200):
        s = DDIMSchedulerB200()
        s.set_timesteps(n)
        x = x_T = torch.linspace(-2.0, 2.0, 9, dtype=torch.float64)
        for t in s.timesteps.tolist():
            x = s.step((1 - ab[t]).sqrt() * x / v(t), t, x).prev_sample
        exact = x_T * (v(0) / v(int(s.timesteps[0]))).sqrt()
        errs.append(float((x - exact).norm() / exact.norm()))
    ratios = [errs[0] / errs[1], errs[1] / errs[2]]
    print(f"DDIM: errors {errs}, ratios per doubling {ratios}")
    assert all(1.6 <= r <= 2.4 for r in ratios), (errs, ratios)


def test_ddim_rows_equal_per_row_schedulers(fake_steps, monkeypatch):
    """PNDMRowsB200 built with the DDIM class: every row equals its own DDIMSchedulerB200 run, bit for bit in fp64,
    with rows starting at 0, in the middle and at the last step; no row pushes history"""
    from test_interpolation_cpu import _fake_pndm_step

    from riffusion import tc_ops
    from riffusion.scheduler_b200 import DDIMSchedulerB200, PNDMRowsB200

    monkeypatch.setattr(tc_ops, "cfg_pndm_step", _fake_pndm_step)      # the definition _fake_rows_step shares

    steps, starts, g = 10, [0, 4, 9], [5.0, 7.0, 9.0]
    rows = PNDMRowsB200(steps, starts, g, device="cpu", scheduler=DDIMSchedulerB200)
    ref = DDIMSchedulerB200()
    ref.set_timesteps(steps)
    assert rows.timesteps.tolist() == ref.timesteps.tolist()
    assert (rows.table["push"] == -1).all() and (rows.table["h1"] == -1).all()
    B = len(g)
    gen = torch.Generator().manual_seed(1)
    x0 = torch.randn((B, 4, 3, 5), generator=gen, dtype=torch.float64)
    pairs = [torch.randn((2 * B, 4, 3, 5), generator=gen, dtype=torch.float64) for _ in range(steps)]
    x = x0
    for j, t in enumerate(rows.timesteps):
        x = rows.step_cfg(pairs[j], 0.0, int(t), x)
    for r in range(B):
        s = DDIMSchedulerB200()
        s.set_timesteps(steps)
        want = x0[r:r + 1]
        for j in range(starts[r], steps):
            want = s.step_cfg(torch.cat([pairs[j][r:r + 1], pairs[j][B + r:B + r + 1]]), g[r], int(s.timesteps[j]), want)
        assert torch.equal(x[r:r + 1], want), r


# ----------------------------------------------------------------------------------------------- Euler ancestral
def test_euler_a_tables():
    from riffusion.scheduler_b200 import EulerAncestralSchedulerB200, make_scheduler

    s = make_scheduler(EA)
    assert isinstance(s, EulerAncestralSchedulerB200) and s.config.get("steps_offset", 0) == 0
    assert abs(s.init_noise_sigma - 14.6146) < 1e-4 and s.init_noise_sigma == float(s.sigmas_full.max())
    s.set_timesteps(50)
    assert s.timesteps.dtype == torch.float64 and len(s.timesteps) == 50
    assert s.timesteps[0] == 999.0 and s.timesteps[-1] == 0.0 and abs(float(s.timesteps[1]) - 978.6122) < 1e-4
    assert s.sigmas.dtype == np.float32 and len(s.sigmas) == 51 and s.sigmas[-1] == 0.0
    assert abs(float(s.sigmas[0]) - 14.6146) < 1e-4 and s.sigmas[0] == s.sigmas_full[999]
    assert np.all(np.diff(s.sigmas) < 0)
    assert s.index(s.timesteps[7].item()) == 7
    with pytest.raises(ValueError, match="not a timestep"):
        s.index(500.0)


def test_euler_a_step_matches_diffusers_form(fake_steps):
    """step_cfg with injected z against the oracle's x0 / derivative / dt / sigma_up form, fp64, to 1e-12;
    scale_model_input and add_noise against the oracle's"""
    from riffusion.scheduler_b200 import EulerAncestralSchedulerB200

    ours, ref = EulerAncestralSchedulerB200(), EulerAncestralOracle()
    n, g = 12, 7.0
    ours.set_timesteps(n)
    ref.set_timesteps(n)
    gen = torch.Generator().manual_seed(0)
    z = torch.randn((n, 2, 4, 3, 5), generator=gen, dtype=torch.float64)
    ours.set_step_noise(z)
    x_o = x_r = torch.randn((2, 4, 3, 5), generator=gen, dtype=torch.float64) * ref.init_noise_sigma
    for k, t in enumerate(ref.timesteps.tolist()):
        assert torch.allclose(ours.scale_model_input(x_o, t), ref.scale_model_input(x_r, t), rtol=1e-7, atol=0)
        pair = torch.randn((4, 4, 3, 5), generator=gen, dtype=torch.float64)
        x_r = ref.step(pair[:2] + g * (pair[2:] - pair[:2]), t, x_r, z[k])
        x_o = ours.step_cfg(pair, g, t, x_o)
        assert torch.allclose(x_o, x_r, rtol=1e-12, atol=1e-12), t
    with pytest.raises(ValueError, match="set_step_noise"):
        ours.step_cfg(pair, g, ref.timesteps[-1].item(), x_o)
    x, nz = torch.randn((2, 4, 3, 5), dtype=torch.float64), torch.randn((2, 4, 3, 5), dtype=torch.float64)
    t = ref.timesteps[3].item()
    # the diffusers-style step draws z from the generator it is given, in the model output's dtype
    got = ours.step(nz, t, x, generator=torch.Generator().manual_seed(5)).prev_sample
    z3 = torch.randn((2, 4, 3, 5), generator=torch.Generator().manual_seed(5), dtype=torch.float64)
    assert torch.allclose(got, ref.step(nz, t, x, z3), rtol=1e-12, atol=1e-12)
    assert torch.allclose(ours.add_noise(x, nz, t), x + ref.sigmas[3].double() * nz, rtol=1e-15, atol=0)


def test_euler_a_weak_convergence_on_gaussian_data(fake_steps):
    """Gaussian data x0 ~ N(0, s^2) with the exact eps(x, sigma) = sigma x / (s^2 + sigma^2): started from
    sigma_max * randn, the ancestral sampler's final variance approaches s^2 with first-order weak error, so
    |var(final) / s^2 - 1| falls ~2x per doubling of n.  400 000 scalar samples (statistical error ~0.002)."""
    from riffusion.scheduler_b200 import EulerAncestralSchedulerB200

    s2, N = 1.0, 400_000
    errs = []
    for n in (80, 160, 320):
        s = EulerAncestralSchedulerB200()
        s.set_timesteps(n)
        rng = np.random.default_rng(0)
        x = torch.from_numpy(rng.standard_normal(N) * s.init_noise_sigma)
        s.set_step_noise(torch.from_numpy(rng.standard_normal((n, N))))
        for i, t in enumerate(s.timesteps.tolist()):
            sig = float(s.sigmas[i])
            eps = sig * x / (s2 + sig * sig)
            x = s.step_cfg(torch.cat([eps, eps]), 0.0, t, x)
        errs.append(abs(float(x.var()) / s2 - 1))
    ratios = [errs[0] / errs[1], errs[1] / errs[2]]
    print(f"Euler ancestral: |var/s^2 - 1| {errs}, ratios per doubling {ratios}")
    assert all(1.6 <= r <= 2.4 for r in ratios), (errs, ratios)


# ----------------------------------------------------------------------------------------------- pipeline
class _RecordingUNet:
    def __init__(self):
        self.inputs, self.ts = [], []

    def __call__(self, x, t, encoder_hidden_states=None, **kw):
        self.inputs.append(x.clone())
        self.ts.append(t)
        out = 0.3 * torch.tanh(x.float()) + 0.002 * (float(t) / 1000.0) + \
            0.05 * encoder_hidden_states.float().mean(dim=(1, 2))[:, None, None, None]
        return types.SimpleNamespace(sample=out.to(torch.float16))


@pytest.fixture
def pipe(monkeypatch, fake_steps):
    from riffusion import scheduler_b200
    from riffusion.riffusion_pipeline import RiffusionPipeline

    noises = []

    def euler_a(eps_pair, guidance, guidance_rows, sample, noise, dt, sigma_up):
        noises.append(noise.clone())
        return _fake_euler_a(eps_pair, guidance, guidance_rows, sample, noise, dt, sigma_up)

    monkeypatch.setattr(scheduler_b200, "cfg_euler_a_step", euler_a)
    unet = _RecordingUNet()
    p = RiffusionPipeline(vae=None, unet=unet, device="cpu")
    p.use_cuda_graph = False
    p.noises = noises
    return p, unet


def _emb():
    torch.manual_seed(4)
    return torch.randn(1, 77, 16).half(), torch.randn(1, 77, 16).half()


def test_txt2img_counts_timesteps_scaling_and_draws(pipe):
    """n evaluations for both schedulers; Euler ancestral hands the UNet its float timesteps and the scaled input,
    scales the initial latents by init_noise_sigma, and steps with z drawn from clip i's generator (seed + i) after its
    latents, one (1, 4, h, w) fp16 draw per step; DDIM draws nothing beyond the latents"""
    from riffusion.scheduler_b200 import EulerAncestralSchedulerB200

    p, unet = pipe
    text, uncond = _emb()
    kw = dict(seed=7, num_clips=3, num_inference_steps=6, width=128, height=64, output_type="latent",
              text_embeddings=text, uncond_embeddings=uncond)
    out = p.txt2img("", scheduler=DDIM, **kw)
    assert out["n_unet_evals"] == 6 == len(unet.inputs) and not p.noises
    assert unet.ts == [166 * k + 1 for k in range(6)][::-1]
    assert all(type(t) is int for t in unet.ts)
    unet.inputs.clear(), unet.ts.clear()
    out = p.txt2img("", scheduler=EA, **kw)
    ref = EulerAncestralSchedulerB200()
    ref.set_timesteps(6)
    assert out["n_unet_evals"] == 6 == len(unet.inputs) == len(p.noises)
    assert unet.ts == ref.timesteps.tolist() and all(type(t) is float for t in unet.ts)
    gens = [torch.Generator().manual_seed(7 + i) for i in range(3)]
    lat = torch.cat([torch.randn((1, 4, 8, 16), generator=g, dtype=torch.float16) for g in gens])
    x = (lat * ref.init_noise_sigma)
    want_in = (x.double() / (float(ref.sigmas[0]) ** 2 + 1) ** 0.5).half()
    assert torch.equal(unet.inputs[0], torch.cat([want_in] * 2))
    for k in range(6):
        want = torch.cat([torch.randn((1, 4, 8, 16), generator=g, dtype=torch.float16) for g in gens])
        assert torch.equal(p.noises[k], want), k
    p.noises.clear()
    z = torch.randn((6, 3, 4, 8, 16)).half()
    p.txt2img("", scheduler=EA, latents=lat, step_noise=z, **{k: v for k, v in kw.items() if k != "seed"})
    assert all(torch.equal(p.noises[k], z[k]) for k in range(6))
    with pytest.raises(ValueError, match="step_noise must be"):
        p.txt2img("", scheduler=EA, step_noise=z[:5], **kw)
    with pytest.raises(ValueError, match="only used by"):
        p.txt2img("", scheduler=DDIM, step_noise=z, **kw)


@pytest.mark.parametrize("scheduler", [DDIM, EA])
def test_img2img_counts_and_draws(pipe, scheduler):
    """13 evaluations at 25 steps and strength 0.55 for both; for Euler ancestral the noise is added at the float
    timestep timesteps[t_start] as x + sigma n, and each image's z stream is its generator (seeded with `seed`) after
    the fp32 posterior draw and the fp16 img2img noise: the same for every image, which one draw serves"""
    from riffusion.riffusion_pipeline import VAE_SCALE

    p, unet = pipe
    text, uncond = _emb()
    mean, logvar = torch.randn(3, 4, 8, 8).half(), (0.1 * torch.randn(3, 4, 8, 8)).half()
    out = p.img2img("", None, moments=(mean, logvar), seed=5, scheduler=scheduler, output_type="latent",
                    text_embeddings=text, uncond_embeddings=uncond)
    assert out["n_unet_evals"] == 13 == len(unet.inputs)
    if scheduler == DDIM:
        assert out["t_start"] == 12 and unet.ts[0] == 481 and not p.noises
        return
    assert out["t_start"] == 12 and len(p.noises) == 13 and type(unet.ts[0]) is float
    for i in range(3):
        g = torch.Generator().manual_seed(5)
        post = torch.randn((1, 4, 8, 8), generator=g)
        std = torch.exp(0.5 * torch.clamp(logvar[i:i + 1], -30.0, 20.0))
        lat = VAE_SCALE * (mean[i:i + 1].float() + std.float() * post).half()
        noise = torch.randn((1, 4, 8, 8), generator=g, dtype=torch.float16)
        for k in range(13):
            assert torch.equal(p.noises[k][i:i + 1], torch.randn((1, 4, 8, 8), generator=g, dtype=torch.float16)), (i, k)
        from riffusion.scheduler_b200 import EulerAncestralSchedulerB200

        s = EulerAncestralSchedulerB200()
        s.set_timesteps(25)
        sig = float(s.sigmas[12])
        x = (lat.double() + sig * noise.double()).half()
        assert torch.equal(unet.inputs[0][i:i + 1], (x.double() / (sig * sig + 1) ** 0.5).half())


def test_ddim_riffuse_and_eta(pipe):
    """interpolate_img2img on a pipeline built with DDIM: 37 evaluations at 50 steps and strength 0.75 over DDIM's
    timesteps; a non-zero eta is refused before any UNet call; Euler ancestral is refused there"""
    from riffusion.scheduler_b200 import DDIMSchedulerB200, EulerAncestralSchedulerB200

    p, unet = pipe
    p.scheduler = DDIMSchedulerB200()
    text, uncond = _emb()
    lat, noise = torch.randn(1, 4, 8, 8).half(), torch.randn(1, 4, 8, 8).half()
    kw = dict(text_embeddings=text, init_latents=lat, generator_a=None, generator_b=None, interpolate_alpha=0.0,
              strength_a=0.75, strength_b=0.75, num_inference_steps=50, guidance_scale=7.0, uncond_embeddings=uncond,
              noise=noise, output_type="latent")
    with pytest.raises(ValueError, match="eta"):
        p.interpolate_img2img(eta=0.3, **kw)
    assert not unet.inputs
    out = p.interpolate_img2img(**kw)
    assert out["n_unet_evals"] == 37 == len(unet.inputs)
    assert unet.ts == [int(t) for t in p.scheduler.timesteps[13:]] and unet.ts[0] == 721 and unet.ts[-1] == 1
    p.scheduler = EulerAncestralSchedulerB200()
    unet.inputs.clear()
    with pytest.raises(ValueError, match="Euler ancestral"):
        p.interpolate_img2img(**kw)
    assert not unet.inputs


def test_magic_mix_refuses_euler_a_before_any_work(pipe, monkeypatch):
    """Euler ancestral is refused by magic_mix and audio_to_audio(magic_mix=True) before any device work; DDIM runs"""
    from riffusion import tc_ops

    monkeypatch.setattr(tc_ops, "magic_mix", lambda x, enc, noise, a, b, mix:
                        (mix * x.double() + (1 - mix) * (a * enc.double() + b * noise.double())).half())
    p, unet = pipe
    text, uncond = _emb()
    moments = (torch.zeros(1, 4, 8, 8).half(), torch.zeros(1, 4, 8, 8).half())
    with pytest.raises(ValueError, match="Magic Mix"):
        p.magic_mix("", None, moments=moments, scheduler=EA, text_embeddings=text, uncond_embeddings=uncond)
    with pytest.raises(ValueError, match="Magic Mix"):
        p.audio_to_audio(types.SimpleNamespace(frame_rate=44100), "", magic_mix=True, scheduler=EA)
    out = p.magic_mix("", None, moments=moments, scheduler=DDIM, num_inference_steps=10, output_type="latent",
                      text_embeddings=text, uncond_embeddings=uncond)
    assert out["n_unet_evals"] == 10 - out["t_max"] == len(unet.inputs)


def test_lms_and_euler_still_refused(pipe):
    from riffusion.scheduler_b200 import make_scheduler
    from riffusion.text_to_audio_batch import parse_batch

    p, unet = pipe
    text, uncond = _emb()
    moments = (torch.zeros(1, 4, 8, 8).half(), torch.zeros(1, 4, 8, 8).half())
    for name in ("LMSDiscreteScheduler", "EulerDiscreteScheduler"):
        match = "supported: DPMSolverMultistepScheduler, PNDMScheduler, DDIMScheduler, EulerAncestralDiscreteScheduler"
        with pytest.raises(ValueError, match=match):
            make_scheduler(name)
        with pytest.raises(ValueError, match="DPMSolverMultistepScheduler, PNDMScheduler"):
            p.txt2img("", scheduler=name, text_embeddings=text, uncond_embeddings=uncond)
        with pytest.raises(ValueError, match="DPMSolverMultistepScheduler, PNDMScheduler"):
            p.img2img("", None, moments=moments, scheduler=name, text_embeddings=text, uncond_embeddings=uncond)
        with pytest.raises(ValueError, match="DPMSolverMultistepScheduler, PNDMScheduler"):
            p.magic_mix("", None, moments=moments, scheduler=name, text_embeddings=text, uncond_embeddings=uncond)
        with pytest.raises(ValueError, match="unsupported scheduler"):
            parse_batch({"params": {"scheduler": name}, "entries": [{"prompt": "a"}]})
    assert not unet.inputs


# ----------------------------------------------------------------------------------------------- batch
FOUR = {"params": [{"name": "dpm", "guidance": 5.0, "num_inference_steps": 4, "width": 64},
                   {"name": "pndm", "scheduler": PNDM, "guidance": 7.0, "num_inference_steps": 4, "width": 64},
                   {"name": "ddim", "scheduler": DDIM, "guidance": 6.0, "num_inference_steps": 5, "width": 64},
                   {"name": "ddim9", "scheduler": DDIM, "guidance": 9.0, "num_inference_steps": 5, "width": 64},
                   {"name": "ea", "scheduler": EA, "guidance": 8.0, "num_inference_steps": 3, "width": 64},
                   {"name": "ea6", "scheduler": EA, "guidance": 6.5, "num_inference_steps": 3, "width": 64}],
        "entries": [{"prompt": "church bells", "seed": 3}, {"prompt": "jazz", "negative_prompt": "drums", "seed": 8}]}


def test_batch_with_all_four_schedulers(batch_pipe, monkeypatch):
    """one loop per scheduler (sets differing only in guidance share it), n evaluations for DDIM and Euler ancestral;
    the Euler-ancestral rows get each row's guidance and z drawn from the row's seed after its latents; every clip
    equals txt2img of its prompt, seed and param set (row-wise fake UNet, so bit for bit)"""
    from riffusion import scheduler_b200, tc_ops
    from riffusion.text_to_audio_batch import parse_batch, plan_batch

    pipe, unet, rows_guidances = batch_pipe
    monkeypatch.setattr(tc_ops, "axpby", _axpby64)
    calls = []

    def euler_a(eps_pair, guidance, guidance_rows, sample, noise, dt, sigma_up):
        calls.append((None if guidance_rows is None else guidance_rows.clone(), noise.clone()))
        return _fake_euler_a(eps_pair, guidance, guidance_rows, sample, noise, dt, sigma_up)

    monkeypatch.setattr(scheduler_b200, "cfg_euler_a_step", euler_a)
    _, loops = plan_batch(*parse_batch(FOUR))
    assert [(lp.scheduler, len(lp.rows), lp.n_unet_evals) for lp in loops] == \
        [(DPM, 2, 4), (PNDM, 2, 5), (DDIM, 4, 5), (EA, 4, 3)]
    out = pipe.text_to_audio_batch(FOUR)
    assert [(lp["scheduler"], lp["n_unet_evals"]) for lp in out["loops"]] == [(DPM, 4), (PNDM, 5), (DDIM, 5), (EA, 3)]
    assert len(unet.inputs) == 4 + 5 + 5 + 3
    clips = out["clips"]
    ea_rows = out["loops"][3]["rows"]
    assert len(calls) == 3 and calls[0][0].tolist() == [8.0 if clips[k]["param_name"] == "ea" else 6.5 for k in ea_rows]
    gens = [torch.Generator().manual_seed(clips[k]["seed"]) for k in ea_rows]
    for g in gens:
        torch.randn((1, 4, 64, 8), generator=g, dtype=torch.float16)
    for k in range(3):
        want = torch.cat([torch.randn((1, 4, 64, 8), generator=g, dtype=torch.float16) for g in gens])
        assert torch.equal(calls[k][1], want), k
    calls.clear()
    for c in clips:
        ps = FOUR["params"][c["param_index"]]
        want = pipe.txt2img(c["prompt"], negative_prompt=c["negative_prompt"], seed=c["seed"],
                            num_inference_steps=ps["num_inference_steps"], guidance_scale=ps["guidance"], width=64,
                            height=512, scheduler=ps.get("scheduler", DPM), output_type="latent")
        assert torch.equal(c["image"], _u8(want["latents"])[0]), (c["entry_index"], c["seed"], c["param_index"])


# ----------------------------------------------------------------------------------------------- operand contract
def _lat(*lead):
    return torch.zeros((*lead, 4, 8, 8), dtype=torch.float16)


def _g(b, dtype=torch.float32, device="cpu"):
    return torch.full((b,), 7.0, dtype=dtype, device=device)


VALID = {
    "scalar": lambda: (_lat(6), 7.0, None, _lat(3), _lat(3), -0.5, 0.3),
    "rows": lambda: (_lat(6), 0.0, _g(3), _lat(3), _lat(3), -0.5, 0.3),
    "no_noise": lambda: (_lat(6), 7.0, None, _lat(3), None, -0.5, 0.0),
}
MALFORMED = {
    "guidance_length": lambda: (_lat(6), 0.0, _g(2), _lat(3), _lat(3), -0.5, 0.3),
    "guidance_dtype": lambda: (_lat(6), 0.0, _g(3, torch.float16), _lat(3), _lat(3), -0.5, 0.3),
    "guidance_2d": lambda: (_lat(6), 0.0, _g(3)[:, None], _lat(3), _lat(3), -0.5, 0.3),
    "eps_pair_rows": lambda: (_lat(3), 7.0, None, _lat(3), _lat(3), -0.5, 0.3),
    "eps_pair_dtype": lambda: (_lat(6).float(), 7.0, None, _lat(3), _lat(3), -0.5, 0.3),
    "noise_shape": lambda: (_lat(6), 7.0, None, _lat(3), _lat(2), -0.5, 0.3),
    "noise_dtype": lambda: (_lat(6), 7.0, None, _lat(3), _lat(3).float(), -0.5, 0.3),
    "noise_strided": lambda: (_lat(6), 7.0, None, _lat(3), _lat(3).transpose(2, 3), -0.5, 0.3),
    "second_device": lambda: (_lat(6), 0.0, _g(3, device="meta"), _lat(3), _lat(3), -0.5, 0.3),
    "sample_dtype": lambda: (_lat(6), 7.0, None, _lat(3).float(), _lat(3), -0.5, 0.3),
    "sample_empty": lambda: (_lat(0), 7.0, None, _lat(0), None, -0.5, 0.3),
}


def test_euler_a_step_contract(recorder):  # noqa: F811
    from riffusion import _native
    from riffusion.scheduler_b200 import cfg_euler_a_step

    for name, run in VALID.items():
        recorder.clear()
        prev = cfg_euler_a_step(*run())
        assert recorder == ["rf_cfg_euler_a_step_f16"], name
        assert prev.shape == (3, 4, 8, 8) and prev.dtype == torch.float16
    for name, run in MALFORMED.items():
        recorder.clear()
        with pytest.raises((ValueError, _native.NativeError)):
            cfg_euler_a_step(*run())
        assert recorder == [], name


def test_euler_a_step_refuses_host_tensors(monkeypatch):
    from riffusion import _native
    from riffusion.scheduler_b200 import cfg_euler_a_step

    calls = []
    monkeypatch.setattr(_native, "call", lambda name, device, *args: calls.append(name))
    with pytest.raises(_native.NativeError, match="CUDA tensor"):
        cfg_euler_a_step(*VALID["scalar"]())
    assert calls == []


# ----------------------------------------------------------------------------------------------- bench
def test_bench_accounting_new_schedulers():
    spec = importlib.util.spec_from_file_location("bench_text_to_audio", ROOT / "tools" / "bench_text_to_audio.py")
    mod = importlib.util.module_from_spec(spec)
    sys.modules["bench_text_to_audio"] = mod
    spec.loader.exec_module(mod)
    assert mod.n_unet_evals(DDIM, 30) == 30 and mod.n_unet_evals(EA, 30) == 30
    with pytest.raises(ValueError):
        mod.n_unet_evals("LMSDiscreteScheduler", 30)
