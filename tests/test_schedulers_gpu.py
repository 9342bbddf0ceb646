"""DDIM and Euler ancestral on the H100: `rf_cfg_euler_a_step_f16` against fp64 and against itself in rows mode, the
txt2img loops of both schedulers against the fp32 oracle loop, the pipeline's Euler-ancestral draws against the CUDA
generator, a text-to-audio batch that mixes all four schedulers against txt2img, and the audio entry points end to end.
The loop bar is that of tests/test_text_to_audio_gpu.py: within 1.3 x the loop's fp16-storage floor + 2e-4."""
import numpy as np
import pytest
import torch

from scheduler_oracle import DDIMOracle, EulerAncestralOracle, loop, loop_emul
from test_audio_to_audio_gpu import _track
from test_parity_bench_gpu import rel_l2
from test_text_to_audio_gpu import _no_tf32, _t2a_pipe, small_unet, vae_pair  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu

DPM, PNDM, DDIM, EA = "DPMSolverMultistepScheduler", "PNDMScheduler", "DDIMScheduler", "EulerAncestralDiscreteScheduler"


# ----------------------------------------------------------------------------------------------- the kernel
@torch.no_grad()
@pytest.mark.parametrize("index", [0, 7, 9])
def test_euler_a_kernel_against_fp64(native_lib, index):
    """the guided eps as torch's fp16 expression, then x' = x + dt eps + sigma_up z within one fp16 rounding + 2^-20
    relative of fp64 from the same fp16 inputs, at sigma-space magnitudes up to 60 (index 9 is the last step: sigma_up 0);
    rows mode gives the scalar kernel's bits at each row's guidance; no noise equals sigma_up = 0"""
    from riffusion.scheduler_b200 import EulerAncestralSchedulerB200, cfg_euler_a_step

    s = EulerAncestralSchedulerB200()
    s.set_timesteps(10)
    dt, up = s.coefficients(s.timesteps[index].item())
    torch.manual_seed(index)
    shape = (4, 3, 7, 13)
    B = shape[0]
    pair = torch.randn((2 * B,) + shape[1:], device="cuda").half()
    x = ((torch.rand(shape, device="cuda") * 2 - 1) * 60).half()
    z = torch.randn(shape, device="cuda").half()
    g = 7.5
    prev = cfg_euler_a_step(pair, g, None, x, z, dt, up)
    eu, et = pair[:B], pair[B:]
    eps = eu + g * (et - eu)                                            # torch fp16 arithmetic
    dt32, up32 = float(np.float32(dt)), float(np.float32(up))
    p64 = x.double() + dt32 * eps.double() + up32 * z.double()
    mag = x.double().abs() + abs(dt32) * eps.double().abs() + abs(up32) * z.double().abs()
    ulp = lambda v: torch.finfo(torch.float16).eps * v.abs().clamp_min(2.0 ** -14)       # noqa: E731
    assert bool(((prev.double() - p64).abs() <= 0.5 * ulp(p64) + 2.0 ** -20 * mag).all())
    # eps alone: x = 0, dt = 1, no noise gives the guided eps exactly
    assert torch.equal(cfg_euler_a_step(pair, g, None, torch.zeros_like(x), None, 1.0, 0.0), eps)
    gr = [7.5, 0.0, 3.25, 12.0]
    rows = cfg_euler_a_step(pair, 0.0, torch.tensor(gr, device="cuda"), x, z, dt, up)
    for r in range(B):
        one = cfg_euler_a_step(torch.cat([pair[r:r + 1], pair[B + r:B + r + 1]]), gr[r], None, x[r:r + 1],
                               z[r:r + 1], dt, up)
        assert torch.equal(rows[r:r + 1], one), r
    assert torch.equal(cfg_euler_a_step(pair, g, None, x, None, dt, up), cfg_euler_a_step(pair, g, None, x, z, dt, 0.0))


# ----------------------------------------------------------------------------------------------- the loops
@torch.no_grad()
@pytest.mark.parametrize("scheduler,steps", [(DDIM, 10), (EA, 10), (EA, 20)])
def test_txt2img_loop_matches_oracle_loop(small_unet, scheduler, steps):
    """txt2img (reduced-width UNet, 16x24 latents, injected latents, embeddings and step noise) against the fp32
    oracle loop; the floor is the fp16-storage loop's distance to it.  Graph replay equals the eager path bit for bit."""
    from riffusion.riffusion_pipeline import RiffusionPipeline

    oracle, ours = small_unet
    pipe = RiffusionPipeline(vae=None, unet=ours, device="cuda")
    torch.manual_seed(steps)
    lat = torch.randn(1, 4, 16, 24, device="cuda").half()
    text = torch.randn(1, 77, 64, device="cuda").half()
    uncond = torch.randn(1, 77, 64, device="cuda").half()
    z = torch.randn(steps, 1, 4, 16, 24, device="cuda").half() if scheduler == EA else None
    kw = dict(num_inference_steps=steps, width=192, height=128, scheduler=scheduler, output_type="latent",
              text_embeddings=text, uncond_embeddings=uncond, latents=lat, step_noise=z)
    out = pipe.txt2img("", **kw)
    mk = DDIMOracle if scheduler == DDIM else EulerAncestralOracle
    zz = None if z is None else z[:, 0].float()
    ref, n_ref = loop(oracle, mk(torch.float32), text.float(), uncond.float(), lat.float(), steps, 7.0, zz)
    emul, n_emul = loop_emul(oracle, mk(), text, uncond, lat, steps, 7.0, zz)
    assert out["n_unet_evals"] == n_ref == n_emul == steps
    e, floor = rel_l2(out["latents_unscaled"], ref), rel_l2(emul, ref)
    print(f"txt2img {scheduler} {steps} steps: rel_l2 {e:.3e}, fp16-storage floor of the loop {floor:.3e}")
    assert e <= 1.3 * floor + 2e-4
    pipe.use_cuda_graph = False
    eager = pipe.txt2img("", **kw)
    assert torch.equal(eager["latents_unscaled"], out["latents_unscaled"])


@torch.no_grad()
def test_euler_a_draws_are_the_cuda_generator_sequence(small_unet):
    """txt2img: clip i's generator (seed + i) draws its latents, then one fp16 tensor per step; img2img: every image's
    generator (seed) draws the fp32 posterior noise, the img2img noise, then one tensor per step.  A call that draws
    equals one with those draws injected, bit for bit."""
    from riffusion.riffusion_pipeline import RiffusionPipeline, _sample_latents

    _, ours = small_unet
    pipe = RiffusionPipeline(vae=None, unet=ours, device="cuda")
    torch.manual_seed(2)
    text = torch.randn(1, 77, 64, device="cuda").half()
    uncond = torch.randn(1, 77, 64, device="cuda").half()
    kw = dict(num_inference_steps=6, scheduler=EA, output_type="latent", text_embeddings=text,
              uncond_embeddings=uncond)
    drawn = pipe.txt2img("", seed=3, num_clips=2, width=192, height=128, **kw)
    gens = [torch.Generator("cuda").manual_seed(3 + i) for i in range(2)]
    lat = torch.cat([torch.randn((1, 4, 16, 24), generator=g, device="cuda", dtype=torch.float16) for g in gens])
    z = torch.stack([torch.cat([torch.randn((1, 4, 16, 24), generator=g, device="cuda", dtype=torch.float16)
                                for g in gens]) for _ in range(6)])
    injected = pipe.txt2img("", num_clips=2, width=192, height=128, latents=lat, step_noise=z, **kw)
    assert torch.equal(drawn["latents_unscaled"], injected["latents_unscaled"])
    mean = torch.randn(2, 4, 16, 24, device="cuda").half()
    logvar = (0.1 * torch.randn(2, 4, 16, 24, device="cuda")).half()
    drawn = pipe.img2img("", None, moments=(mean, logvar), seed=9, **kw)
    assert drawn["n_unet_evals"] == 6 - drawn["t_start"]
    n_run = drawn["n_unet_evals"]
    noises, zs = [], []
    for i in range(2):
        g = torch.Generator("cuda").manual_seed(9)
        _sample_latents(mean[i:i + 1], logvar[i:i + 1], g)
        noises.append(torch.randn((1, 4, 16, 24), generator=g, device="cuda", dtype=torch.float16))
        zs.append(torch.cat([torch.randn((1, 4, 16, 24), generator=g, device="cuda", dtype=torch.float16)
                             for _ in range(n_run)]))
    assert torch.equal(zs[0], zs[1])
    injected = pipe.img2img("", None, moments=(mean, logvar), seed=9, noise=torch.cat(noises),
                            step_noise=torch.stack(zs, dim=1), **kw)
    assert torch.equal(drawn["latents_unscaled"], injected["latents_unscaled"])


# ----------------------------------------------------------------------------------------------- batch
@torch.no_grad()
def test_batch_mixing_all_four_schedulers(vae_pair):
    """one text-to-audio batch with a DPM-Solver++, a PNDM, a DDIM and an Euler-ancestral param set over two seeds:
    every clip's latents equal txt2img of the same two clips (the same batch composition), bit for bit"""
    _, vae = vae_pair
    pipe = _t2a_pipe(vae)
    params = [{"name": s[:4], "scheduler": s, "guidance": 7.0, "num_inference_steps": 4, "width": 64}
              for s in (DPM, PNDM, DDIM, EA)]
    batch = {"params": params, "entries": [{"prompt": "church bells", "seed": 3}, {"prompt": "church bells", "seed": 4}]}
    out = pipe.text_to_audio_batch(batch, apply_filters=False)
    assert [lp["scheduler"] for lp in out["loops"]] == [DPM, PNDM, DDIM, EA]
    assert [lp["n_unet_evals"] for lp in out["loops"]] == [4, 5, 4, 4]
    for p, s in enumerate((DPM, PNDM, DDIM, EA)):
        want = pipe.txt2img("church bells", seed=3, num_clips=2, num_inference_steps=4, guidance_scale=7.0, width=64,
                            height=512, scheduler=s, output_type="latent")["latents_unscaled"]
        got = [c for c in out["clips"] if c["param_index"] == p]
        assert [c["seed"] for c in got] == [3, 4]
        for j, c in enumerate(got):
            assert torch.equal(c["latents_unscaled"], want[j]), (s, j)
            assert torch.isfinite(c["waveform"]).all()


# ----------------------------------------------------------------------------------------------- end to end
@torch.no_grad()
@pytest.mark.parametrize("scheduler", [DDIM, EA])
def test_text_to_audio_and_cli(vae_pair, tmp_path, monkeypatch, scheduler):
    """text_to_audio and `python -m riffusion.cli text-to-audio --scheduler ...` write finite audio of the expected
    length"""
    from riffusion import cli
    from riffusion.riffusion_pipeline import RiffusionPipeline
    from riffusion.util.audio_util import AudioSegment

    _, vae = vae_pair
    pipe = _t2a_pipe(vae)
    out = pipe.text_to_audio("church bells", seed=5, num_inference_steps=5, width=256, scheduler=scheduler)
    assert out["n_unet_evals"] == 5 and out["waveform"].shape == (1, 1, 441 * 255)
    assert torch.isfinite(out["waveform"]).all() and out["waveform"].abs().max() > 0
    monkeypatch.setattr(RiffusionPipeline, "load_checkpoint", classmethod(lambda cls, **kw: pipe))
    cli.main(["text-to-audio", "--prompt", "jazz", "--audio", str(tmp_path / "o.wav"), "--width", "256",
              "--num-inference-steps", "4", "--scheduler", scheduler])
    seg = AudioSegment.from_file(str(tmp_path / "o.wav"))
    a = np.asarray(seg.get_array_of_samples())
    assert seg.channels == 1 and abs(seg.duration_seconds - 441 * 255 / 44100) < 1e-3 and np.abs(a).max() > 0


@torch.no_grad()
@pytest.mark.parametrize("scheduler", [DDIM, EA])
def test_audio_to_audio(vae_pair, scheduler):
    """audio_to_audio at its defaults (25 steps, denoising 0.55) runs 13 evaluations per batch and gives finite audio"""
    _, vae = vae_pair
    pipe = _t2a_pipe(vae)
    out = pipe.audio_to_audio(_track(), "church bells", seed=5, scheduler=scheduler)
    assert out["n_unet_evals"] == [13]
    assert torch.isfinite(out["waveform"]).all() and abs(out["segment"].duration_seconds - 9.8) < 1e-3
