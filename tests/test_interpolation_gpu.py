"""Interpolation on the H100: `rf_cfg_pndm_rows_step_f16` against fp64 and against `rf_cfg_pndm_step_f16`, the walk
against `riffuse_batch` and `riffuse`, graph replay, batching, the stitched track and the `interpolation` command."""
import numpy as np
import pytest
import torch
from PIL import Image

from test_text_to_audio_gpu import _t2a_pipe, vae_pair  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu


def _table(B, recs):
    from riffusion.scheduler_b200 import ROW_DTYPE

    t = np.zeros(B, dtype=ROW_DTYPE)
    for name in ("h1", "h2", "h3", "push"):
        t[name] = -1
    for r, rec in enumerate(recs):
        for k, v in rec.items():
            t[r][k] = v
    return torch.from_numpy(t.view(np.int32).reshape(B, -1)).cuda()


def _guided(eps_pair, g, B):
    """torch's fp16 guidance combine with a per-row guidance: (et - eu) rounded, * g rounded, + eu rounded"""
    eu, et = eps_pair[:B], eps_pair[B:]
    d = et - eu
    gd = (d.float() * torch.tensor(g, dtype=torch.float32, device="cuda").view(B, 1, 1, 1)).half()
    return eu + gd


@torch.no_grad()
def test_rows_kernel_against_fp64(native_lib):
    """random records: inactive rows, a first step that saves its sample, a restart from the saved sample, 1- to
    4-term combinations, per-row guidance; an odd element count per row"""
    from riffusion.scheduler_b200 import ROW_BASE_SAVED, ROW_SAVE, cfg_pndm_rows_step

    torch.manual_seed(11)
    shape = (7, 4, 9, 13)
    B = shape[0]
    pair = torch.randn((2 * B,) + shape[1:], device="cuda").half()
    x = (torch.randn(shape, device="cuda") * 2).half()
    ring = torch.randn((4,) + shape, device="cuda").half()
    saved = torch.randn(shape, device="cuda").half()
    g = [7.0, 3.5, 0.0, 9.25, 1.75, 5.0, 12.0]
    recs = [
        dict(active=0, guidance=g[0]),
        dict(active=1, guidance=g[1], c0=1.0, ca=0.97, cb=0.11, push=0, flags=ROW_SAVE),
        dict(active=1, guidance=g[2], c0=0.5, c1=0.5, h1=2, ca=1.02, cb=0.2, flags=ROW_BASE_SAVED),
        dict(active=1, guidance=g[3], c0=1.5, c1=-0.5, h1=3, ca=0.99, cb=0.05, push=1),
        dict(active=1, guidance=g[4], c0=23 / 12, c1=-16 / 12, c2=5 / 12, h1=0, h2=1, ca=1.01, cb=0.3, push=2),
        dict(active=1, guidance=g[5], c0=55 / 24, c1=-59 / 24, c2=37 / 24, c3=-9 / 24, h1=3, h2=2, h3=0, ca=0.95,
             cb=0.07, push=1),
        dict(active=0, guidance=g[6], push=3, flags=ROW_SAVE),
    ]
    ring0, saved0 = ring.clone(), saved.clone()
    prev = cfg_pndm_rows_step(pair, _table(B, recs), ring, saved, x)
    e0 = _guided(pair, g, B)
    for r, rec in enumerate(recs):
        if not rec["active"]:
            assert torch.equal(prev[r], x[r]) and torch.equal(ring[:, r], ring0[:, r]) and torch.equal(saved[r], saved0[r])
            continue
        f = lambda v: float(np.float32(v))          # noqa: E731  (the C floats the kernel reads)
        e = f(rec["c0"]) * e0[r].double()
        for c, h in (("c1", "h1"), ("c2", "h2"), ("c3", "h3")):
            if rec.get(h, -1) >= 0:
                e = e + f(rec[c]) * ring0[rec[h], r].double()
        base = saved0[r] if rec.get("flags", 0) & ROW_BASE_SAVED else x[r]
        want = f(rec["ca"]) * base.double() - f(rec["cb"]) * e
        err = (prev[r].double() - want).abs()
        tol = want.abs() * 2 ** -11 + 1e-6 * (want.abs().max() + 1)
        assert (err <= tol).all(), (r, float(err.max()))
        if rec.get("push", -1) >= 0:
            assert torch.equal(ring[rec["push"]][r], e0[r])
        for s in range(4):
            if s != rec.get("push", -1):
                assert torch.equal(ring[s][r], ring0[s][r]), (r, s)
        assert torch.equal(saved[r], x[r] if rec.get("flags", 0) & ROW_SAVE else saved0[r])


@torch.no_grad()
def test_homogeneous_table_is_the_single_step_kernel(native_lib):
    """every row holding one PNDMSchedulerB200 step gives rf_cfg_pndm_step_f16's bits, for each kind of step"""
    from riffusion import tc_ops
    from riffusion.scheduler_b200 import ROW_BASE_SAVED, cfg_pndm_rows_step

    torch.manual_seed(12)
    shape = (5, 4, 16, 16)
    B = shape[0]
    pair = torch.randn((2 * B,) + shape[1:], device="cuda").half()
    x = torch.randn(shape, device="cuda").half()
    hist = [torch.randn(shape, device="cuda").half() for _ in range(3)]
    saved = torch.randn(shape, device="cuda").half()
    ca, cb = 0.9983, 0.0421
    for coef, n_hist, restart in (((1.0, 0, 0, 0), 0, False), ((0.5, 0.5, 0, 0), 1, True), ((1.5, -0.5, 0, 0), 1, False),
                                  ((23 / 12, -16 / 12, 5 / 12, 0), 2, False),
                                  ((55 / 24, -59 / 24, 37 / 24, -9 / 24), 3, False)):
        ring = torch.zeros((4,) + shape, device="cuda").half()
        slots = [3, 1, 0][:n_hist]
        for s, h in zip(slots, hist):
            ring[s] = h
        rec = dict(active=1, guidance=7.5, c0=coef[0], c1=coef[1], c2=coef[2], c3=coef[3], ca=ca, cb=cb, push=2,
                   flags=ROW_BASE_SAVED if restart else 0)
        rec.update({h: s for h, s in zip(("h1", "h2", "h3"), slots)})
        prev = cfg_pndm_rows_step(pair, _table(B, [rec] * B), ring, saved.clone(), x)
        eps, want = tc_ops.cfg_pndm_step(pair, 7.5, hist[:n_hist], coef, saved if restart else x, ca, cb)
        assert torch.equal(prev, want), coef
        assert torch.equal(ring[2], eps), coef


# ----------------------------------------------------------------------------------------------- the walk
def _seed_image(width=256, seed=0):
    """a smooth random 512-high image (mono 0-10 kHz spectrograms have 512 frequency rows)"""
    rng = np.random.default_rng(seed)
    base = rng.integers(0, 256, (512 // 8, width // 8, 3), dtype=np.uint8)
    return Image.fromarray(base).resize((width, 512), Image.BICUBIC)


def _ends(den_a, den_b, g_a=7.0, g_b=7.0):
    from riffusion.datatypes import PromptInput

    return (PromptInput(prompt="church bells", seed=3, denoising=den_a, guidance=g_a),
            PromptInput(prompt="jazz (piano:1.2)", seed=8, denoising=den_b, guidance=g_b))


def _close(a, b, what):
    d = np.abs(np.asarray(a).astype(np.int16) - np.asarray(b).astype(np.int16))
    print(f"{what}: mean |diff| {d.mean():.4f} LSB, max {d.max()}, within 1 LSB {(d <= 1).mean():.4f}")
    assert d.mean() < 0.25 and (d <= 1).mean() >= 0.98, what


@torch.no_grad()
def test_one_group_walk_is_riffuse_batch(vae_pair):
    """alphas 0, 0.5, 1 with equal ends are one riffuse_batch group: the walk gives its images bit for bit"""
    _, vae = vae_pair
    pipe = _t2a_pipe(vae)
    start, end = _ends(0.75, 0.75)
    img = _seed_image()
    out = pipe.interpolation(start, end, img, num_interpolation_steps=3, num_inference_steps=10)
    assert out["alphas"].tolist() == [0.0, 0.5, 1.0] and out["n_unet_evals"] == [8]
    want = pipe.riffuse_batch(out["requests"], img)
    for i in range(3):
        assert np.array_equal(out["images"][i].cpu().numpy(), np.asarray(want[i])), i


@torch.no_grad()
def test_heterogeneous_walk_rows_are_riffuse_graph_and_batching(vae_pair):
    """a 0.5 -> 0.9 walk with guidance 7 -> 5: one loop whose rows join at their own start; each row against `riffuse` of
    its request; graph replay is eager bit for bit; max_batch=2 against the default"""
    _, vae = vae_pair
    pipe = _t2a_pipe(vae)
    start, end = _ends(0.5, 0.9, 7.0, 5.0)
    img = _seed_image(seed=1)
    kw = dict(num_interpolation_steps=4, num_inference_steps=10)
    out = pipe.interpolation(start, end, img, **kw)
    assert out["n_unet_evals"] == [10]
    for i, req in enumerate(out["requests"]):
        _close(out["images"][i].cpu().numpy(), pipe.riffuse(req, img), f"walk row {i} vs riffuse")
    pipe.use_cuda_graph = False
    eager = pipe.interpolation(start, end, img, **kw)
    pipe.use_cuda_graph = True
    assert torch.equal(eager["images"], out["images"])
    two = pipe.interpolation(start, end, img, max_batch=2, **kw)
    assert len(two["n_unet_evals"]) == 2
    _close(two["images"].cpu().numpy(), out["images"].cpu().numpy(), "max_batch=2 vs default")
    assert np.abs(out["images"][0].cpu().numpy().astype(np.int16) - out["images"][3].cpu().numpy()).mean() > 0.5


@torch.no_grad()
def test_stitched_track_is_the_per_image_audio(vae_pair):
    """the segment is each image's waveform (the device tail of `_u8_to_waveform` with the same initial phases),
    peak-normalised, filtered and appended without a crossfade: n clips long"""
    from riffusion.riffusion_pipeline import DEFAULT_PARAMS
    from riffusion.util import audio_util

    _, vae = vae_pair
    pipe = _t2a_pipe(vae)
    start, end = _ends(0.6, 0.8)
    img = _seed_image(seed=2)
    conv = pipe._converter(DEFAULT_PARAMS, None)
    n, frames = 3, 256
    angles = torch.rand((n, 1, DEFAULT_PARAMS.n_fft // 2 + 1, frames), dtype=torch.complex64, device="cuda")
    out = pipe.interpolation(start, end, img, num_interpolation_steps=n, num_inference_steps=8, init_angles=angles)
    assert out["images"].shape == (n, 512, 256, 3)
    wave = pipe._u8_to_waveform(out["images"], conv, False, angles)
    assert torch.equal(wave, out["waveform"])
    segs = [audio_util.apply_filters(audio_util.audio_from_waveform(samples=w, sample_rate=44100, normalize=True))
            for w in wave.cpu().numpy()]
    want = np.concatenate([np.asarray(s.get_array_of_samples()) for s in segs])
    got = np.asarray(out["segment"].get_array_of_samples())
    assert np.array_equal(got, want)
    assert len(got) == n * DEFAULT_PARAMS.hop_length * (frames - 1)


def test_interpolation_cli(vae_pair, tmp_path, monkeypatch):
    """`interpolation` end to end with the checkpoint loader replaced by the reduced pipeline"""
    from riffusion import cli
    from riffusion.riffusion_pipeline import DEFAULT_PARAMS, RiffusionPipeline
    from riffusion.spectrogram_params import SpectrogramParams
    from riffusion.util.audio_util import AudioSegment

    _, vae = vae_pair
    pipe = _t2a_pipe(vae)
    monkeypatch.setattr(RiffusionPipeline, "load_checkpoint", classmethod(lambda cls, **kw: pipe))
    _seed_image(seed=3).save(tmp_path / "seed.png")
    cli.main(["interpolation", "--prompt-a", "jazz", "--prompt-b", "rock", "--seed-image", str(tmp_path / "seed.png"),
              "--output", str(tmp_path / "walk.wav"), "--image-dir", str(tmp_path / "img"),
              "--num-interpolation-steps", "2", "--num-inference-steps", "6", "--denoising-b", "0.9"])
    seg = AudioSegment.from_file(str(tmp_path / "walk.wav"))
    assert seg.frame_rate == 44100 and abs(seg.duration_seconds - 2 * 441 * 255 / 44100) < 1e-3
    for i in range(2):
        img = Image.open(tmp_path / "img" / f"step_{i}.png")
        assert img.size == (256, 512) and SpectrogramParams.from_exif(img.getexif()) == DEFAULT_PARAMS
    torch.cuda.synchronize()
