"""Magic Mix on the H100: rf_magic_mix_f16 against fp64, magic_mix loops against an fp32 oracle loop (a literal
restatement of the algorithm on the fp32 UNet oracle, below; the algorithm is unpinned: diffusers' community pipeline
restated from memory), graph replay / batching, audio_to_audio(magic_mix=True) end to end and the `audio-to-audio
--magic-mix` command.

Bars are those of tests/test_parity_bench_gpu.py: loops within 1.3 x the fp16-storage floor of the loop (+2e-4)."""
import numpy as np
import pytest
import torch

from test_audio_to_audio_gpu import _moments, _params, _track
from test_parity_bench_gpu import rel_l2
from test_text_to_audio_gpu import _no_tf32, _t2a_pipe, small_unet, vae_pair  # noqa: F401  (fixtures)
from txt2img_oracle import DPMSolverMultistepOracle

pytestmark = pytest.mark.gpu

DPM, PNDM = "DPMSolverMultistepScheduler", "PNDMScheduler"


# ----------------------------------------------------------------------------------------------- oracle loops
def magic_mix_loop(unet, sched, text, uncond, enc, noise, steps, kmin, kmax, mix, guidance):
    """Magic Mix in fp32: x = add_noise(enc, noise, T[t_max]), then for i >= t_max one CFG evaluation of u and one step
    of x, u = mix x + (1 - mix) add_noise(enc, noise, T[i]) for t_max < i < t_min, else x.  Returns (x, evaluations)."""
    sched.set_timesteps(steps)
    ts = [int(t) for t in sched.timesteps]
    t_min, t_max = steps - int(kmin * steps), steps - int(kmax * steps)
    ctx = torch.cat([uncond, text])

    def add_noise(t):
        a = sched.alphas_cumprod[t]
        return a.sqrt() * enc + (1 - a).sqrt() * noise

    x = add_noise(ts[t_max])
    for i in range(t_max, len(ts)):
        u = mix * x + (1 - mix) * add_noise(ts[i]) if t_max < i < t_min else x
        eu, et = unet(torch.cat([u, u]), ts[i], ctx).chunk(2)
        x = sched.step(eu + guidance * (et - eu), ts[i], x)
    return x, len(ts) - t_max


@torch.no_grad()
def magic_mix_loop_emul(unet_module, sched, text, uncond, enc, noise, steps, kmin, kmax, mix, guidance):
    """magic_mix_loop with fp16 storage where the device path stores fp16: the UNet (oracle.unet_emul), u and the
    noising rounded once from the fp32 noise (rf_magic_mix_f16), the guided eps as three fp16 ops, and the rounding
    points of the step kernels (PNDM: one rounding of the next sample; DPM-Solver++: x0 and the next sample rounded once
    each, as tests/img2img_oracle.py's img2img_loop_emul).  Its distance to the fp32 loop is the fp16-storage floor."""
    from oracle import unet_emul as ue
    from oracle import unet_oracle as uo

    s = sched
    s.set_timesteps(steps)
    ts = [int(t) for t in s.timesteps]
    t_min, t_max = steps - int(kmin * steps), steps - int(kmax * steps)
    ctx = torch.cat([uncond, text]).float()
    f32 = lambda v: float(np.float32(v))                                   # noqa: E731
    enc, noise = ue.r16(enc.float()), noise.float()

    def add_noise(t):
        a = float(s.alphas_cumprod[t])
        return f32(a ** 0.5) * enc + f32((1.0 - a) ** 0.5) * noise

    x = ue.r16(add_noise(ts[t_max]))
    pndm = isinstance(s, uo.PNDMSchedulerOracle)
    ab = s.alphas_cumprod.double()
    a64, sg64 = ab.sqrt(), (1 - ab).sqrt()
    l64 = a64.log() - sg64.log()
    m1 = None
    for j, i in enumerate(range(t_max, len(ts))):
        t = ts[i]
        u = ue.r16(f32(mix) * x + f32(1 - f32(mix)) * add_noise(t)) if t_max < i < t_min else x
        eu, et = ue.unet_forward(unet_module, torch.cat([u, u]), t, ctx).chunk(2)
        e0 = ue.r16(eu + ue.r16(ue.r16(et - eu) * guidance))
        if pndm:
            x = ue.r16(s.step(e0, t, x))
            continue
        prev = 0 if i == len(ts) - 1 else ts[i + 1]
        final = i == len(ts) - 1 and s.lower_order_final and len(ts) < 15
        order = 1 if (s.solver_order == 1 or j == 0 or final) else 2
        h = float(l64[prev] - l64[t])
        x0 = ue.r16((x - f32(sg64[t]) * e0) / f32(a64[t]))
        nxt = f32(sg64[prev] / sg64[t]) * x + f32(-float(a64[prev]) * np.expm1(-h)) * x0
        if order == 2:
            r0 = float(l64[t] - l64[ts[i - 1]]) / h
            nxt = nxt + f32(0.5 * (-float(a64[prev]) * np.expm1(-h)) / r0) * (x0 - m1)
        x, m1 = ue.r16(nxt), x0
    return x, len(ts) - t_max


def _scheduler_oracle(name):
    from oracle import unet_oracle as uo

    return DPMSolverMultistepOracle() if name == DPM else uo.PNDMSchedulerOracle()


def _enc_and_noise(mean, logvar, seed):
    """what magic_mix draws: each image's posterior sample from a CUDA generator seeded with `seed`, and one fp32 CPU
    draw torch.randn((1, 4, h, w)) after seeding with `seed`"""
    from riffusion.riffusion_pipeline import VAE_SCALE
    from riffusion.vae_b200 import _Posterior

    enc = torch.cat([VAE_SCALE * _Posterior(mean[i:i + 1], logvar[i:i + 1]).sample(
        generator=torch.Generator(device="cuda").manual_seed(seed)) for i in range(mean.shape[0])])
    noise = torch.randn((1,) + tuple(mean.shape[1:]), generator=torch.Generator().manual_seed(seed))
    return enc, noise.cuda()


# ----------------------------------------------------------------------------------------------- K1
@pytest.mark.parametrize("shape", [(3, 4, 17, 23), (1, 1, 1, 7), (2, 4, 64, 65)])
@pytest.mark.parametrize("mix", [0.0, 0.3, 1.0])
def test_magic_mix_kernel(native_lib, shape, mix):
    """u within one fp16 rounding + 2^-20 relative of an fp64 evaluation on the fp32 scalars the kernel receives (odd
    element counts); mix = 1 returns x bit for bit, signed zeros included"""
    from riffusion import tc_ops
    from riffusion.scheduler_b200 import DPMSolverMultistepSchedulerB200

    torch.manual_seed(sum(shape) + int(10 * mix))
    x = (torch.randn(shape, device="cuda") * 2).half()
    x.view(-1)[0] = -0.0
    enc = (torch.randn(shape, device="cuda") * 0.8).half()
    noise = torch.randn(shape, device="cuda")
    s = DPMSolverMultistepSchedulerB200()
    ab = float(s.alphas_cumprod[601])
    a, b = ab ** 0.5, (1.0 - ab) ** 0.5
    u = tc_ops.magic_mix(x, enc, noise, a, b, mix)
    assert u.dtype == torch.float16 and u.shape == x.shape
    if mix == 1.0:
        assert torch.equal(u.view(torch.int16), x.view(torch.int16))
        return
    m = np.float32(mix)
    w, a32, b32 = float(np.float32(1.0) - m), float(np.float32(a)), float(np.float32(b))
    xd, ed, nd = x.double(), enc.double(), noise.double()
    u64 = float(m) * xd + w * (a32 * ed + b32 * nd)
    mag = abs(float(m)) * xd.abs() + w * (a32 * ed.abs() + b32 * nd.abs())
    ulp = torch.finfo(torch.float16).eps * u64.abs().clamp_min(2.0 ** -14)
    err = (u.double() - u64).abs()
    assert bool((err <= 0.5 * ulp + 2.0 ** -20 * mag).all()), float((err - 0.5 * ulp).max())


# ----------------------------------------------------------------------------------------------- K2
@torch.no_grad()
@pytest.mark.parametrize("scheduler,steps,kmin,kmax", [(DPM, 25, 0.3, 0.5), (PNDM, 25, 0.3, 0.5), (DPM, 10, 0.2, 0.8)])
def test_magic_mix_loop_matches_oracle_loop(small_unet, scheduler, steps, kmin, kmax):
    """magic_mix (reduced-width UNet, 16x24 latents, injected moments and embeddings) against magic_mix_loop on the fp32
    oracle from the same draws; the floor is magic_mix_loop_emul's distance to it"""
    from riffusion.riffusion_pipeline import RiffusionPipeline

    oracle, ours = small_unet
    pipe = RiffusionPipeline(vae=None, unet=ours, device="cuda")
    torch.manual_seed(steps)
    text = torch.randn(1, 77, 64, device="cuda").half()
    uncond = torch.randn(1, 77, 64, device="cuda").half()
    mean, logvar = _moments(1, 13)
    kw = dict(kmin=kmin, kmax=kmax, num_inference_steps=steps, seed=21, scheduler=scheduler, output_type="latent",
              text_embeddings=text, uncond_embeddings=uncond, moments=(mean, logvar))
    out = pipe.magic_mix("", None, **kw)
    enc, noise = _enc_and_noise(mean, logvar, 21)
    injected = pipe.magic_mix("", None, noise=noise, **kw)
    assert torch.equal(out["latents_unscaled"], injected["latents_unscaled"])        # the CPU fp32 draw
    args = (text.float(), uncond.float(), enc.float(), noise, steps, kmin, kmax, 0.5, 7.0)
    ref, n_ref = magic_mix_loop(oracle, _scheduler_oracle(scheduler), *args)
    emul, n_emul = magic_mix_loop_emul(oracle, _scheduler_oracle(scheduler), text, uncond, enc, noise, steps, kmin,
                                       kmax, 0.5, 7.0)
    want = {(DPM, 25): 12, (PNDM, 25): 13, (DPM, 10): 8}[(scheduler, steps)]
    assert out["n_unet_evals"] == n_ref == n_emul == want
    e, floor = rel_l2(out["latents_unscaled"], ref), rel_l2(emul, ref)
    print(f"magic_mix {scheduler} {steps} steps kmin {kmin} kmax {kmax}: rel_l2 {e:.3e}, fp16-storage floor of the loop "
          f"{floor:.3e}")
    assert e <= 1.3 * floor + 2e-4


# ----------------------------------------------------------------------------------------------- K3
@torch.no_grad()
def test_magic_mix_graph_and_batch(small_unet):
    """graph replay equals the eager path bit for bit; image i of a batch of 3 equals a single-image call within
    sqrt(2) x the loop bar"""
    from riffusion.riffusion_pipeline import RiffusionPipeline

    oracle, ours = small_unet
    pipe = RiffusionPipeline(vae=None, unet=ours, device="cuda")
    torch.manual_seed(8)
    text = torch.randn(1, 77, 64, device="cuda").half()
    uncond = torch.randn(1, 77, 64, device="cuda").half()
    mean, logvar = _moments(3, 9)
    kw = dict(kmin=0.3, kmax=0.6, num_inference_steps=12, seed=4, output_type="latent", text_embeddings=text,
              uncond_embeddings=uncond)
    graphed = pipe.magic_mix("", None, moments=(mean, logvar), **kw)
    assert (graphed["t_max"], graphed["t_min"]) == (5, 9)
    pipe.use_cuda_graph = False
    eager = pipe.magic_mix("", None, moments=(mean, logvar), **kw)
    pipe.use_cuda_graph = True
    assert torch.equal(graphed["latents_unscaled"], eager["latents_unscaled"])
    enc, noise = _enc_and_noise(mean, logvar, 4)
    ref, _ = magic_mix_loop(oracle, DPMSolverMultistepOracle(), text.float(), uncond.float(), enc[:1].float(), noise,
                            12, 0.3, 0.6, 0.5, 7.0)
    emul, _ = magic_mix_loop_emul(oracle, DPMSolverMultistepOracle(), text, uncond, enc[:1], noise, 12, 0.3, 0.6, 0.5,
                                  7.0)
    floor = rel_l2(emul, ref)
    for i in range(3):
        single = pipe.magic_mix("", None, moments=(mean[i:i + 1], logvar[i:i + 1]), **kw)
        e = rel_l2(graphed["latents_unscaled"][i:i + 1], single["latents_unscaled"])
        print(f"magic_mix image {i}: batch of 3 vs single call {e:.3e} (fp16-storage floor of the loop {floor:.3e})")
        assert e <= 2 ** 0.5 * (1.3 * floor + 2e-4), (i, e, floor)


# ----------------------------------------------------------------------------------------------- K4
@torch.no_grad()
def test_audio_to_audio_magic_mix(vae_pair):
    """audio_to_audio(magic_mix=True) on a two-clip track: 5 evaluations per batch at 10 steps, source images as in the
    img2img mode, a different riff from img2img, and max_batch=1 within the fp16 floor of the default"""
    _, vae = vae_pair
    pipe = _t2a_pipe(vae)
    track = _track()
    angles = torch.rand(2, 1, 8821, 501, dtype=torch.complex64, device="cuda", generator=torch.Generator("cuda").manual_seed(2))
    kw = dict(params=_params(False), num_inference_steps=10, seed=5, init_angles=angles)
    out = pipe.audio_to_audio(track, "church bells on sunday", magic_mix=True, **kw)
    assert out["n_unet_evals"] == [5] and np.allclose(out["clip_start_times"], [0.0, 4.8])
    assert out["images"].shape == (2, 512, 501, 3) and out["segment"].channels == 1
    plain = pipe.audio_to_audio(track, "church bells on sunday", **kw)
    assert torch.equal(plain["source_images"], out["source_images"])
    assert (plain["denoised_images"].float() - out["denoised_images"].float()).abs().mean() > 0.5
    one = pipe.audio_to_audio(track, "church bells on sunday", magic_mix=True, max_batch=1, **kw)
    assert one["n_unet_evals"] == [5, 5]
    d = np.abs(one["images"].cpu().numpy().astype(np.int16) - out["images"].cpu().numpy().astype(np.int16))
    print(f"audio_to_audio magic_mix max_batch=1 vs 2: mean |diff| {d.mean():.4f} LSB, max {d.max()}")
    assert d.mean() < 0.25 and (d <= 1).mean() > 0.98


def test_audio_to_audio_magic_mix_cli(vae_pair, tmp_path, monkeypatch):
    """`audio-to-audio --magic-mix` end to end with the checkpoint loader replaced by the reduced pipeline"""
    from PIL import Image

    from riffusion import cli
    from riffusion.riffusion_pipeline import RiffusionPipeline
    from riffusion.util.audio_util import AudioSegment

    _, vae = vae_pair
    pipe = _t2a_pipe(vae)
    monkeypatch.setattr(RiffusionPipeline, "load_checkpoint", classmethod(lambda cls, **kw: pipe))
    _track().export(str(tmp_path / "in.wav"), format="wav")
    cli.main(["audio-to-audio", "--audio", str(tmp_path / "in.wav"), "--output", str(tmp_path / "out.wav"), "--prompt",
              "jazz with piano", "--image-dir", str(tmp_path / "img"), "--num-inference-steps", "6", "--magic-mix",
              "--kmin", "0.2", "--kmax", "0.6", "--mix-factor", "0.4", "--scheduler", PNDM])
    seg = AudioSegment.from_file(str(tmp_path / "out.wav"))
    assert seg.frame_rate == 44100 and seg.channels == 1 and abs(seg.duration_seconds - 9.8) < 1e-3
    for i in range(2):
        assert Image.open(tmp_path / "img" / f"clip_{i}_riffed.png").size == (501, 512)
    torch.cuda.synchronize()
