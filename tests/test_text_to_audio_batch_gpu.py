"""Text to audio batch on the H100: `rf_cfg_dpmpp_rows_step_f16` against fp64 and against `rf_cfg_dpmpp_step_f16`, the
batched loops against txt2img and against the fp32 oracle loop per row, the device tail, and the `text-to-audio-batch`
command.  The loop bar is that of tests/test_text_to_audio_gpu.py: within 1.3 x the loop's fp16-storage floor + 2e-4."""
import json
from pathlib import Path

import numpy as np
import pytest
import torch
from PIL import Image

from test_parity_bench_gpu import rel_l2
from test_text_to_audio_gpu import _no_tf32, _t2a_pipe, small_unet, vae_pair  # noqa: F401  (fixtures)
from txt2img_oracle import DPMSolverMultistepOracle, txt2img_loop, txt2img_loop_emul

pytestmark = pytest.mark.gpu

DPM, PNDM = "DPMSolverMultistepScheduler", "PNDMScheduler"


def _guided(pair, g, B):
    """torch's fp16 guidance combine with a per-row guidance: (et - eu) rounded, * g rounded, + eu rounded"""
    eu, et = pair[:B], pair[B:]
    gd = ((et - eu).float() * torch.tensor(g, dtype=torch.float32, device="cuda").view(B, 1, 1, 1)).half()
    return eu + gd


def _coefs(second_order, index=5):
    from riffusion.scheduler_b200 import DPMSolverMultistepSchedulerB200

    sched = DPMSolverMultistepSchedulerB200()
    sched.set_timesteps(30)
    sched.lower_order_nums = 1 if second_order else 0
    order, coefs = sched.plan(int(sched.timesteps[index]))
    assert order == (2 if second_order else 1)
    return coefs


# ----------------------------------------------------------------------------------------------- the rows kernel
@torch.no_grad()
@pytest.mark.parametrize("second_order", [False, True])
def test_rows_kernel_against_fp64(native_lib, second_order):
    """per-row guidance including 0 and 1, an odd element count per row (3 x 7 x 13); guided eps bit-identical to
    torch's fp16 expression, x0 and x' within one fp16 rounding + 2^-20 relative of fp64, as test_cfg_dpmpp_step_kernel"""
    from riffusion.scheduler_b200 import cfg_dpmpp_rows_step

    torch.manual_seed(41 + second_order)
    shape = (5, 3, 7, 13)
    B = shape[0]
    g = [7.5, 0.0, 3.25, 12.0, 1.0]
    pair = torch.randn((2 * B,) + shape[1:], device="cuda").half()
    x = (torch.randn(shape, device="cuda") * 3).half()
    m1 = torch.randn(shape, device="cuda").half() if second_order else None
    coefs = _coefs(second_order)
    x0, prev = cfg_dpmpp_rows_step(pair, torch.tensor(g, device="cuda"), x, m1, coefs)
    eps = _guided(pair, g, B)
    a, s, c_x, c_0, c_1 = (float(np.float32(v)) for v in coefs)
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
    # sigma = -1, alpha = 1, x = 0: x0 is the guided eps itself, bit for bit
    x0e, _ = cfg_dpmpp_rows_step(pair, torch.tensor(g, device="cuda"), torch.zeros_like(x), None,
                                 (1.0, -1.0, 1.0, 0.0, 0.0))
    assert torch.equal(x0e, eps)


@torch.no_grad()
@pytest.mark.parametrize("second_order", [False, True])
def test_rows_kernel_is_the_scalar_kernel(native_lib, second_order):
    """row r gives rf_cfg_dpmpp_step_f16's bits at g[r]; a uniform guidance gives its bits over the whole batch"""
    from riffusion import tc_ops
    from riffusion.scheduler_b200 import cfg_dpmpp_rows_step

    torch.manual_seed(43 + second_order)
    shape = (4, 4, 64, 65)
    B = shape[0]
    pair = torch.randn((2 * B,) + shape[1:], device="cuda").half()
    x = torch.randn(shape, device="cuda").half()
    m1 = torch.randn(shape, device="cuda").half() if second_order else None
    coefs = _coefs(second_order, 9)
    g = [5.0, 7.0, 9.0, 0.0]
    x0, prev = cfg_dpmpp_rows_step(pair, torch.tensor(g, device="cuda"), x, m1, coefs)
    for r in range(B):
        x0_r, prev_r = tc_ops.cfg_dpmpp_step(torch.cat([pair[r:r + 1], pair[B + r:B + r + 1]]), g[r], x[r:r + 1],
                                             None if m1 is None else m1[r:r + 1], coefs)
        assert torch.equal(x0[r:r + 1], x0_r) and torch.equal(prev[r:r + 1], prev_r), r
    x0, prev = cfg_dpmpp_rows_step(pair, torch.full((B,), 7.5, device="cuda"), x, m1, coefs)
    x0_s, prev_s = tc_ops.cfg_dpmpp_step(pair, 7.5, x, m1, coefs)
    assert torch.equal(x0, x0_s) and torch.equal(prev, prev_s)


# ----------------------------------------------------------------------------------------------- the loops
def _embedder(dim, seed=0):
    """seeded (1, 77, dim) fp16 embeddings per text, in place of a text encoder"""
    cache = {}

    def embed(text):
        if text not in cache:
            g = torch.Generator().manual_seed(seed + len(cache) + 1)
            cache[text] = torch.randn((1, 77, dim), generator=g).half().cuda()
        return cache[text]

    return embed


def _draw(seed, width):
    return torch.randn((1, 4, 64, width // 8), generator=torch.Generator("cuda").manual_seed(seed), device="cuda",
                       dtype=torch.float16)


ENTRIES = [{"prompt": "church bells", "seed": 3}, {"prompt": "jazz", "negative_prompt": "drums", "seed": 8},
           {"prompt": "violin", "seed": 11}]


@torch.no_grad()
@pytest.mark.parametrize("scheduler", [DPM, PNDM])
def test_one_param_set_is_txt2img(small_unet, vae_pair, scheduler):
    """one param set: one loop at the batch size of the entries, bit-identical to txt2img with the same per-row
    embeddings and draws, and its images are the decode of those latents"""
    from riffusion.riffusion_pipeline import RiffusionPipeline

    _, ours = small_unet
    _, vae = vae_pair
    pipe = RiffusionPipeline(vae=vae, unet=ours, device="cuda")
    pipe.embed_text = _embedder(64)
    batch = {"params": {"scheduler": scheduler, "num_inference_steps": 6, "guidance": 7.0, "width": 128},
             "entries": ENTRIES}
    out = pipe.text_to_audio_batch(batch)
    assert [lp["rows"] for lp in out["loops"]] == [[0, 1, 2]]
    assert out["loops"][0]["n_unet_evals"] == (6 if scheduler == DPM else 7)
    texts = torch.cat([pipe.embed_text(e["prompt"]) for e in ENTRIES])
    unconds = torch.cat([pipe.embed_text(e.get("negative_prompt") or "") for e in ENTRIES])
    want = pipe.txt2img("", num_clips=3, num_inference_steps=6, guidance_scale=7.0, width=128, height=512,
                        scheduler=scheduler, output_type="latent", text_embeddings=texts, uncond_embeddings=unconds,
                        latents=torch.cat([_draw(e["seed"], 128) for e in ENTRIES]))
    got = torch.stack([c["latents_unscaled"] for c in out["clips"]])
    assert torch.equal(got, want["latents_unscaled"])
    assert torch.equal(torch.stack([c["image"] for c in out["clips"]]), pipe._decode_u8(want["latents"]))


@torch.no_grad()
def test_mixed_guidance_loops_match_oracle_per_row(small_unet, vae_pair):
    """a DPM-Solver++ loop at guidance 5 / 9, a PNDM loop at 4 / 8 and a DPM-Solver++ loop at 1 / 0.5: each row within
    the loop bar of txt2img_loop on the fp32 oracle at that row's guidance (1 for rows at or below 1, where txt2img runs
    the text branch alone); the device tail: waveforms of 441 (W - 1) samples, images the decode of the loop's latents"""
    from oracle import unet_oracle as uo
    from riffusion.riffusion_pipeline import VAE_SCALE, RiffusionPipeline

    oracle, ours = small_unet
    _, vae = vae_pair
    pipe = RiffusionPipeline(vae=vae, unet=ours, device="cuda")
    pipe.embed_text = _embedder(64, seed=10)
    W = 128
    sets = [(DPM, 5.0), (DPM, 9.0), (PNDM, 4.0), (PNDM, 8.0), (DPM, 1.0), (DPM, 0.5)]
    batch = {"params": [{"scheduler": s, "guidance": g, "num_inference_steps": 8, "width": W} for s, g in sets],
             "entries": ENTRIES[:2]}
    out = pipe.text_to_audio_batch(batch)
    assert [(lp["scheduler"], len(lp["rows"]), lp["n_unet_evals"]) for lp in out["loops"]] == \
        [(DPM, 4, 8), (PNDM, 4, 9), (DPM, 4, 8)]
    for c in out["clips"]:
        scheduler, g = sets[c["param_index"]]
        e = ENTRIES[c["entry_index"]]
        text, uncond = pipe.embed_text(e["prompt"]), pipe.embed_text(e.get("negative_prompt") or "")
        mk = DPMSolverMultistepOracle if scheduler == DPM else uo.PNDMSchedulerOracle
        g_eff = g if g > 1.0 else 1.0
        lat = _draw(c["seed"], W)
        ref, _ = txt2img_loop(oracle, mk(), text.float(), uncond.float(), lat.float(), 8, g_eff)
        emul, _ = txt2img_loop_emul(oracle, mk(), text, uncond, lat, 8, g_eff)
        err, floor = rel_l2(c["latents_unscaled"][None], ref), rel_l2(emul, ref)
        print(f"{scheduler} guidance {g} entry {c['entry_index']}: rel_l2 {err:.3e}, floor {floor:.3e}")
        assert err <= 1.3 * floor + 2e-4, (scheduler, g, c["entry_index"], err, floor)
        assert c["waveform"].shape == (1, 441 * (W - 1)) and torch.isfinite(c["waveform"]).all()
        assert c["image"].shape == (512, W, 3) and c["image"].dtype == torch.uint8
    for lp in out["loops"]:
        lat = torch.stack([out["clips"][k]["latents_unscaled"] for k in lp["rows"]])
        u8 = pipe._decode_u8((1.0 / VAE_SCALE) * lat)
        assert torch.equal(torch.stack([out["clips"][k]["image"] for k in lp["rows"]]), u8)


# ----------------------------------------------------------------------------------------------- the command
def test_text_to_audio_batch_cli(vae_pair, tmp_path, monkeypatch):
    """three entries x two param sets x --num-seeds 2: 12 image / audio pairs with the seed in their names, 1.27 s each
    at width 128, EXIF params that round-trip, and an index.json listing every output"""
    from riffusion import cli
    from riffusion.riffusion_pipeline import DEFAULT_PARAMS, RiffusionPipeline
    from riffusion.spectrogram_params import SpectrogramParams
    from riffusion.util.audio_util import AudioSegment

    _, vae = vae_pair
    pipe = _t2a_pipe(vae)
    monkeypatch.setattr(RiffusionPipeline, "load_checkpoint", classmethod(lambda cls, **kw: pipe))
    data = {"params": [{"name": "g5", "guidance": 5.0, "num_inference_steps": 3, "width": 128},
                       {"name": "g9", "guidance": 9.0, "num_inference_steps": 3, "width": 128}],
            "entries": ENTRIES}
    (tmp_path / "in.json").write_text(json.dumps(data))
    out = tmp_path / "out"
    cli.main(["text-to-audio-batch", "--json", str(tmp_path / "in.json"), "--output-dir", str(out), "--num-seeds", "2"])
    stems = ["church_bells_neg_", "jazz_neg_drums", "violin_neg_"]
    n = 0
    for e, stem in zip(ENTRIES, stems):
        for seed in (e["seed"], e["seed"] + 1):
            for i in range(2):
                img = Image.open(out / f"image_{i}_{stem}_{seed}.jpg")
                assert img.size == (128, 512) and SpectrogramParams.from_exif(img.getexif()) == DEFAULT_PARAMS
                seg = AudioSegment.from_file(str(out / f"audio_{i}_{stem}_{seed}.wav"))
                assert seg.frame_rate == 44100 and seg.channels == 1 and abs(seg.duration_seconds - 1.27) < 1e-3
                n += 1
    assert n == 12 and len(list(out.iterdir())) == 25
    index = json.loads((out / "index.json").read_text())
    outputs = [o for e in index["entries"] for o in e["outputs"]]
    assert len(outputs) == 12 and all(Path(o["image_path"]).exists() and Path(o["audio_path"]).exists() for o in outputs)
    assert [(o["name"], o["seed"]) for o in index["entries"][2]["outputs"]] == \
        [("g5", 11), ("g9", 11), ("g5", 12), ("g9", 12)]
    torch.cuda.synchronize()

