"""Text to audio batch without a GPU: parsing of the batch JSON and its refusals, the clip order and the loop plan, the
DPM-Solver++ rows scheduler against per-row schedulers, the pipeline's control flow with the device steps replaced by
their torch definitions, the operand contract of `cfg_dpmpp_rows_step`, the `text-to-audio-batch` command and the bench
script's accounting."""
import copy
import importlib.util
import json
import sys
import types
from pathlib import Path

import numpy as np
import pytest
import torch
from PIL import Image

from test_op_contracts_cpu import recorder  # noqa: F401  (fixture)

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "tests" / "golden"))

DPM, PNDM = "DPMSolverMultistepScheduler", "PNDMScheduler"
EXAMPLE = {
    "params": {"checkpoint": "riffusion/riffusion-model-v1", "scheduler": DPM, "num_inference_steps": 50,
               "guidance": 7.0, "width": 512},
    "entries": [{"prompt": "Church bells", "seed": 42}, {"prompt": "electronic beats", "negative_prompt": "drums",
                                                         "seed": 100}, {"prompt": "classical violin concerto", "seed": 4}],
}


# ----------------------------------------------------------------------------------------------- parsing
def test_parse_defaults_single_and_list_params():
    from riffusion import text_to_audio_batch as tab

    ps, entries = tab.parse_batch({"params": {}, "entries": [{"prompt": "a"}]})
    assert ps == [tab.ParamSet(name="params[0]", checkpoint="riffusion/riffusion-model-v1", scheduler=DPM,
                               num_inference_steps=50, guidance=7.0, width=512)]
    assert entries == [tab.Entry(prompt="a", negative_prompt=None, seed=42)]
    ps, entries = tab.parse_batch(EXAMPLE)
    assert len(ps) == 1 and ps[0].name == "params[0]" and [e.seed for e in entries] == [42, 100, 4]
    assert entries[1].negative_prompt == "drums"
    ps, _ = tab.parse_batch({"params": [{"guidance": 5}, {"name": "hi", "guidance": 9.0, "scheduler": PNDM,
                                                           "width": 768, "num_inference_steps": 20}, {}],
                             "entries": [{"prompt": "a"}]})
    assert [p.name for p in ps] == ["params[0]", "hi", "params[2]"]
    assert [p.guidance for p in ps] == [5.0, 9.0, 7.0] and isinstance(ps[0].guidance, float)
    assert (ps[1].scheduler, ps[1].width, ps[1].num_inference_steps) == (PNDM, 768, 20)


REFUSALS = {
    "no_params": ({"entries": [{"prompt": "a"}]}, "no 'params'"),
    "no_entries": ({"params": {}}, "no 'entries'"),
    "empty_entries": ({"params": {}, "entries": []}, "non-empty"),
    "no_prompt": ({"params": {}, "entries": [{"seed": 3}]}, "no prompt"),
    "width_not_64": ({"params": {"width": 500}, "entries": [{"prompt": "a"}]}, "multiple of 64"),
    "width_zero": ({"params": {"width": 0}, "entries": [{"prompt": "a"}]}, "multiple of 64"),
    "steps_zero": ({"params": {"num_inference_steps": 0}, "entries": [{"prompt": "a"}]}, "at least 1"),
    "lms": ({"params": {"scheduler": "LMSDiscreteScheduler"}, "entries": [{"prompt": "a"}]}, "unsupported scheduler"),
    "euler": ({"params": [{}, {"scheduler": "EulerDiscreteScheduler"}], "entries": [{"prompt": "a"}]},
              "unsupported scheduler"),
    "param_key": ({"params": {"guidance_scale": 9.0}, "entries": [{"prompt": "a"}]}, "'guidance_scale'"),
    "entry_key": ({"params": {}, "entries": [{"prompt": "a", "sed": 4}]}, "'sed'"),
    "top_key": ({"params": {}, "entries": [{"prompt": "a"}], "num_seeds": 2}, "'num_seeds'"),
    "seed_type": ({"params": {}, "entries": [{"prompt": "a", "seed": "4"}]}, "integer"),
}


@pytest.mark.parametrize("name", list(REFUSALS))
def test_parse_refusals(name):
    from riffusion.text_to_audio_batch import parse_batch

    data, match = REFUSALS[name]
    with pytest.raises(ValueError, match=match):
        parse_batch(data)


def test_module_example_is_valid_json():
    """the module docstring ships a valid example (the app's has a trailing comma)"""
    from riffusion import text_to_audio_batch as tab

    doc = tab.__doc__
    text = doc[doc.index("    {"):doc.index("\n    }\n") + 6]
    ps, entries = tab.parse_batch(json.loads(text))
    assert [p.guidance for p in ps] == [5.0, 7.0] and len(entries) == 3


def test_index_json_parses_back():
    from riffusion import text_to_audio_batch as tab

    data = {"params": [{"guidance": 5.0}, {"name": "g9", "guidance": 9.0}], "entries": EXAMPLE["entries"]}
    ps, entries = tab.parse_batch(data)
    clips, _ = tab.plan_batch(ps, entries, num_seeds=2)
    paths = [(f"i{k}.jpg", f"a{k}.wav") for k in range(len(clips))]
    index = tab.build_index(data, ps, clips, paths)
    assert "outputs" not in data["entries"][0] and "name" not in data["params"][0]      # the input is not changed
    assert [p["name"] for p in index["params"]] == ["params[0]", "g9"]
    e0 = index["entries"][0]
    assert [(o["name"], o["seed"]) for o in e0["outputs"]] == [("params[0]", 42), ("g9", 42), ("params[0]", 43),
                                                               ("g9", 43)]
    assert (e0["image_path"], e0["audio_path"]) == ("i3.jpg", "a3.wav")
    back_ps, back_entries = tab.parse_batch(json.loads(json.dumps(index)))
    assert back_ps == ps and back_entries == entries


# ----------------------------------------------------------------------------------------------- planning
def test_plan_clip_order_grouping_and_chunking():
    """entry, then seed, then param set; groups by (scheduler, steps, width, guidance > 1) in order of first appearance,
    chunked at max_batch in clip order; sets differing only in guidance share a loop"""
    from riffusion.text_to_audio_batch import parse_batch, plan_batch

    data = {"params": [{"guidance": 5.0}, {"guidance": 9.0}, {"guidance": 1.0}, {"scheduler": PNDM, "guidance": 7.0},
                       {"width": 768}],
            "entries": [{"prompt": "a", "seed": 10}, {"prompt": "b", "seed": 3}]}
    ps, entries = parse_batch(data)
    clips, loops = plan_batch(ps, entries, num_seeds=2, max_batch=32)
    assert [(c.entry_index, c.seed, c.param_index) for c in clips[:6]] == \
        [(0, 10, 0), (0, 10, 1), (0, 10, 2), (0, 10, 3), (0, 10, 4), (0, 11, 0)]
    assert len(clips) == 2 * 2 * 5 and clips[-1] == type(clips[0])(param_index=4, entry_index=1, seed=4)
    keys = [(lp.scheduler, lp.width, lp.cfg) for lp in loops]
    assert keys == [(DPM, 512, True), (DPM, 512, False), (PNDM, 512, True), (DPM, 768, True)]
    assert [clips[k].param_index for k in loops[0].rows] == [0, 1] * 4
    assert list(loops[0].rows) == sorted(loops[0].rows)
    assert [lp.n_unet_evals for lp in loops] == [50, 50, 51, 50]
    assert sorted(k for lp in loops for k in lp.rows) == list(range(len(clips)))
    _, small = plan_batch(ps, entries, num_seeds=2, max_batch=3)
    assert [len(lp.rows) for lp in small] == [3, 3, 2, 3, 1, 3, 1, 3, 1]
    assert [k for lp in small[:3] for k in lp.rows] == list(loops[0].rows)
    for kw, match in ((dict(num_seeds=0), "num_seeds"), (dict(max_batch=0), "max_batch")):
        with pytest.raises(ValueError, match=match):
            plan_batch(ps, entries, **kw)


def test_evaluation_counts():
    from riffusion.text_to_audio_batch import n_unet_evals

    assert [n_unet_evals(DPM, n) for n in (1, 25, 50)] == [1, 25, 50]
    assert [n_unet_evals(PNDM, n) for n in (2, 25, 50)] == [3, 26, 51]
    assert n_unet_evals(PNDM, 1) == 1                     # one step has no duplicated PLMS timestep


def test_bench_accounting():
    spec = importlib.util.spec_from_file_location("bench_text_to_audio_batch",
                                                  ROOT / "tools" / "bench_text_to_audio_batch.py")
    mod = importlib.util.module_from_spec(spec)
    sys.modules["bench_text_to_audio_batch"] = mod
    spec.loader.exec_module(mod)
    acc = mod.schedule_accounting(mod.default_batch())
    assert acc == {"clips": 12, "batch": {"loops": 1, "unet_evals": 50, "row_evals": 600},
                   "per_set": {"loops": 3, "unet_evals": 150, "row_evals": 600},
                   "app": {"loops": 12, "unet_evals": 600, "row_evals": 600}}
    acc = mod.schedule_accounting(mod.default_batch(), num_seeds=2, max_batch=5)
    assert acc["batch"] == {"loops": 5, "unet_evals": 250, "row_evals": 1200}
    assert acc["per_set"] == {"loops": 6, "unet_evals": 300, "row_evals": 1200}


# ----------------------------------------------------------------------------------------------- rows scheduler
def _fake_dpm_rows(eps_pair, guidance_rows, sample, m1, coefs):
    """torch definition of rf_cfg_dpmpp_rows_step_f16 in the dtype of the inputs: the scalar step, row r at g[r]"""
    from test_text_to_audio_cpu import _fake_dpm_step

    g = guidance_rows.to(sample.dtype).view(-1, *[1] * (sample.dim() - 1))
    return _fake_dpm_step(eps_pair, g, sample, m1, coefs)


@pytest.mark.parametrize("steps", [10, 20])
def test_dpm_rows_equal_per_row_schedulers(monkeypatch, steps):
    """DPMSolverRowsB200 runs the parent's plan and x0 history: every row equals its own
    DPMSolverMultistepSchedulerB200 run at its guidance, bit for bit in fp64"""
    from test_text_to_audio_cpu import _fake_dpm_step

    from riffusion import scheduler_b200, tc_ops
    from riffusion.scheduler_b200 import DPMSolverMultistepSchedulerB200, DPMSolverRowsB200

    monkeypatch.setattr(tc_ops, "cfg_dpmpp_step", _fake_dpm_step)
    monkeypatch.setattr(scheduler_b200, "cfg_dpmpp_rows_step", _fake_dpm_rows)
    g = [5.0, 7.0, 9.0, 7.5]
    rows = DPMSolverRowsB200(steps, g, device="cpu")
    assert rows.guidance.dtype == torch.float32 and rows.guidance.tolist() == g
    B = len(g)
    gen = torch.Generator().manual_seed(steps)
    x0 = torch.randn((B, 4, 3, 5), generator=gen, dtype=torch.float64)
    pairs = [torch.randn((2 * B, 4, 3, 5), generator=gen, dtype=torch.float64) for _ in range(steps)]
    x = x0
    for j, t in enumerate(rows.timesteps):
        x = rows.step_cfg(pairs[j], 0.0, int(t), x)
    for r in range(B):
        s = DPMSolverMultistepSchedulerB200()
        s.set_timesteps(steps)
        want = x0[r:r + 1]
        for j, t in enumerate(s.timesteps):
            want = s.step_cfg(torch.cat([pairs[j][r:r + 1], pairs[j][B + r:B + r + 1]]), g[r], int(t), want)
        assert torch.equal(x[r:r + 1], want), r


def test_rows_guidance_tables():
    from riffusion.scheduler_b200 import DPMSolverRowsB200, PNDMRowsB200, rows_guidance

    assert rows_guidance([5, 9.5]) == [5.0, 9.5]
    assert rows_guidance([1.0, 0.5]) == [0.0, 0.0]
    assert DPMSolverRowsB200(10, [1.0, 0.0], device="cpu").guidance.tolist() == [0.0, 0.0]
    for make in (lambda g: DPMSolverRowsB200(10, g, device="cpu"), lambda g: PNDMRowsB200(10, [0] * len(g), g, "cpu")):
        with pytest.raises(ValueError, match="both sides of 1"):
            make([7.0, 1.0])
    with pytest.raises(ValueError, match="one guidance per row"):
        DPMSolverRowsB200(10, [], device="cpu")


# ----------------------------------------------------------------------------------------------- pipeline
def _u8(scaled):
    return (scaled.float() * 40 + 128).clamp(0, 255).to(torch.uint8)[:, :3].permute(0, 2, 3, 1).contiguous()


@pytest.fixture
def batch_pipe(monkeypatch):
    """the recording UNet and fake steps of test_audio_to_audio_cpu, the rows steps replaced by their torch
    definitions, the stub text encoder, and host stand-ins for the VAE and the audio tail"""
    from prompt_stub import StubTextEncoder, StubTokenizer
    from test_audio_to_audio_cpu import _pipe
    from test_interpolation_cpu import _fake_pndm_step, _fake_rows_step

    from riffusion import scheduler_b200, tc_ops

    pipe, unet = _pipe(monkeypatch)
    monkeypatch.setattr(tc_ops, "cfg_pndm_step", _fake_pndm_step)    # the fp64 definition _fake_rows_step shares
    rows_guidances = []

    def dpm_rows(eps_pair, guidance_rows, sample, m1, coefs):
        rows_guidances.append(guidance_rows.clone())
        x0, prev = _fake_dpm_rows(eps_pair.float(), guidance_rows, sample.float(), None if m1 is None else m1.float(),
                                  coefs)
        return x0.half(), prev.half()

    def pndm_rows(eps_pair, rows, ring, saved, sample):
        rows_guidances.append(torch.from_numpy(rows.numpy().copy().view(scheduler_b200.ROW_DTYPE)["guidance"][:, 0]))
        return _fake_rows_step(eps_pair, rows, ring, saved, sample)

    monkeypatch.setattr(scheduler_b200, "cfg_dpmpp_rows_step", dpm_rows)
    monkeypatch.setattr(scheduler_b200, "cfg_pndm_rows_step", pndm_rows)
    pipe.text_encoder, pipe.tokenizer = StubTextEncoder(), StubTokenizer()
    pipe._decode_u8 = _u8
    pipe._converter = lambda params, converter: None
    pipe._u8_to_waveform = lambda u8, conv, stereo, angles: \
        torch.sin(u8.float().mean(dim=(1, 3))[:, None, :].repeat(1, 1, 50) / 9.0)
    return pipe, unet, rows_guidances


BATCH = {"params": [{"name": "g5", "guidance": 5.0, "num_inference_steps": 6, "width": 64},
                    {"name": "g9", "guidance": 9.0, "num_inference_steps": 6, "width": 64},
                    {"name": "p", "scheduler": PNDM, "guidance": 7.0, "num_inference_steps": 4, "width": 64},
                    {"name": "low", "guidance": 1.0, "num_inference_steps": 3, "width": 64}],
         "entries": [{"prompt": "church bells", "seed": 3}, {"prompt": "jazz", "negative_prompt": "drums", "seed": 8}]}


def test_pipeline_control_flow(batch_pipe):
    """latents are each row's seeded draw, the context is [negative or "" | prompt] per row, the guidance table holds
    each row's guidance (0 below 1), one UNet call per timestep of each loop; every clip equals txt2img of its prompt,
    negative prompt, seed and param set (row-wise fake UNet, so bit for bit)"""
    pipe, unet, rows_guidances = batch_pipe
    out = pipe.text_to_audio_batch(BATCH, num_seeds=2)
    assert len(out["clips"]) == 2 * 2 * 4
    assert [(lp["scheduler"], len(lp["rows"]), lp["n_unet_evals"]) for lp in out["loops"]] == \
        [(DPM, 8, 6), (PNDM, 4, 5), (DPM, 4, 3)]
    assert len(unet.inputs) == 6 + 5 + 3
    assert [x.shape[0] for x in unet.inputs] == [16] * 6 + [8] * 5 + [4] * 3
    rows0 = out["loops"][0]["rows"]
    clips = out["clips"]
    for j, k in enumerate(rows0):
        c = clips[k]
        draw = torch.randn((1, 4, 64, 8), generator=torch.Generator().manual_seed(c["seed"]), dtype=torch.float16)
        assert torch.equal(unet.inputs[0][j:j + 1], draw) and torch.equal(unet.inputs[0][8 + j:9 + j], draw)
    assert rows_guidances[0].tolist() == [clips[k]["param_name"] == "g9" and 9.0 or 5.0 for k in rows0]
    assert rows_guidances[6].tolist() == [7.0] * 4            # the PNDM loop's first step
    assert rows_guidances[-1].tolist() == [0.0] * 4           # the guidance-1 loop
    assert unet.inputs[-1].shape[0] == 4                      # no CFG doubling below guidance 1
    assert [(c["entry_index"], c["seed"], c["param_index"]) for c in clips[:5]] == \
        [(0, 3, 0), (0, 3, 1), (0, 3, 2), (0, 3, 3), (0, 4, 0)]
    for c in clips:
        ps = BATCH["params"][c["param_index"]]
        assert c["param_name"] == ps["name"]
        assert c["image"].shape == (64, 8, 3) and c["waveform"].shape == (1, 400)
        assert abs(c["segment"].duration_seconds - 400 / 44100) < 1e-9
        want = pipe.txt2img(c["prompt"], negative_prompt=c["negative_prompt"], seed=c["seed"],
                            num_inference_steps=ps["num_inference_steps"], guidance_scale=ps["guidance"], width=64,
                            height=512, scheduler=ps.get("scheduler", DPM), output_type="latent")
        assert torch.equal(c["image"], _u8(want["latents"])[0]), (c["entry_index"], c["seed"], c["param_index"])


def test_pipeline_context_rows(batch_pipe, monkeypatch):
    """the loop's context is [embed_text(negative or "") per row | embed_text(prompt) per row]"""
    pipe, unet, _ = batch_pipe
    seen = []
    real = pipe._context
    monkeypatch.setattr(pipe, "_context", lambda *a: seen.append(a) or real(*a))
    pipe.text_to_audio_batch({"params": BATCH["params"][:2], "entries": BATCH["entries"]})
    (_, _, n, do_cfg, texts, unconds), = seen
    assert n == 4 and do_cfg
    for j, (prompt, neg) in enumerate([("church bells", ""), ("church bells", ""), ("jazz", "drums"),
                                       ("jazz", "drums")]):
        assert torch.equal(texts[j:j + 1], pipe.embed_text(prompt))
        assert torch.equal(unconds[j:j + 1], pipe.embed_text(neg))


def test_pipeline_refusals_before_any_unet_call(batch_pipe):
    pipe, unet, _ = batch_pipe
    for batch, kw, match in ((REFUSALS["lms"][0], {}, "unsupported scheduler"),
                             (REFUSALS["param_key"][0], {}, "guidance_scale"),
                             (BATCH, dict(num_seeds=0), "num_seeds"), (BATCH, dict(max_batch=0), "max_batch")):
        with pytest.raises(ValueError, match=match):
            pipe.text_to_audio_batch(batch, **kw)
    assert not unet.inputs


# ----------------------------------------------------------------------------------------------- operand contract
def _lat(*lead):
    return torch.zeros((*lead, 4, 8, 8), dtype=torch.float16)


def _g(b, dtype=torch.float32, device="cpu"):
    return torch.full((b,), 7.0, dtype=dtype, device=device)


COEFS = (0.9, 0.4, 1.0, 0.1, 0.05)
ROWS_VALID = lambda: (_lat(6), _g(3), _lat(3), _lat(3), COEFS)           # noqa: E731
ROWS_MALFORMED = {
    "guidance_length": lambda: (_lat(6), _g(2), _lat(3), _lat(3), COEFS),
    "guidance_dtype": lambda: (_lat(6), _g(3, torch.float16), _lat(3), _lat(3), COEFS),
    "guidance_2d": lambda: (_lat(6), _g(3)[:, None], _lat(3), _lat(3), COEFS),
    "eps_pair_rows": lambda: (_lat(3), _g(3), _lat(3), _lat(3), COEFS),
    "m1_shape": lambda: (_lat(6), _g(3), _lat(3), _lat(2), COEFS),
    "m1_dtype": lambda: (_lat(6), _g(3), _lat(3), _lat(3).float(), COEFS),
    "second_device": lambda: (_lat(6), _g(3, device="meta"), _lat(3), _lat(3), COEFS),
    "sample_dtype": lambda: (_lat(6), _g(3), _lat(3).float(), _lat(3), COEFS),
    "sample_empty": lambda: (_lat(0), _g(0), _lat(0), None, COEFS),
}


def test_rows_step_contract(recorder):  # noqa: F811
    from riffusion import _native
    from riffusion.scheduler_b200 import cfg_dpmpp_rows_step

    x0, prev = cfg_dpmpp_rows_step(*ROWS_VALID())
    assert recorder == ["rf_cfg_dpmpp_rows_step_f16"]
    assert x0.shape == prev.shape == (3, 4, 8, 8) and prev.dtype == torch.float16
    recorder.clear()
    cfg_dpmpp_rows_step(_lat(6), _g(3), _lat(3), None, COEFS)                  # first order: no m1
    assert recorder == ["rf_cfg_dpmpp_rows_step_f16"]
    for name, run in ROWS_MALFORMED.items():
        recorder.clear()
        with pytest.raises((ValueError, _native.NativeError)):
            cfg_dpmpp_rows_step(*run())
        assert recorder == [], name


def test_rows_step_refuses_host_tensors(monkeypatch):
    from riffusion import _native
    from riffusion.scheduler_b200 import cfg_dpmpp_rows_step

    calls = []
    monkeypatch.setattr(_native, "call", lambda name, device, *args: calls.append(name))
    with pytest.raises(_native.NativeError, match="CUDA tensor"):
        cfg_dpmpp_rows_step(*ROWS_VALID())
    assert calls == []


# ----------------------------------------------------------------------------------------------- CLI
def test_cli_flags_and_registration():
    from riffusion import cli

    sub = next(a for a in cli.build_parser()._actions if a.dest == "command")
    assert len(sub.choices) == 6 and "text-to-audio-batch" not in sub.choices
    assert [f.__name__ for f in cli.BATCH_COMMANDS] == ["text_to_audio_batch"]
    parser = cli.build_parser(cli.COMMANDS + cli.EXTRA_COMMANDS + cli.TRACK_COMMANDS + cli.BATCH_COMMANDS)
    sub = next(a for a in parser._actions if a.dest == "command")
    flags = {o for act in sub.choices["text-to-audio-batch"]._actions for o in act.option_strings}
    assert {"--json", "--output-dir", "--num-seeds", "--max-batch", "--audio-extension", "--checkpoint",
            "--device"} <= flags
    with pytest.raises(SystemExit):
        parser.parse_args(["text-to-audio-batch", "--json", "in.json"])
    ns = parser.parse_args(["text-to-audio-batch", "--json", "in.json", "--output-dir", "out"])
    assert (ns.num_seeds, ns.max_batch, ns.audio_extension, ns.checkpoint, ns.device) == \
        (1, 32, "wav", "riffusion/riffusion-model-v1", "cuda")


def test_cli_writes_files_and_index(monkeypatch, tmp_path, capsys):
    from riffusion import cli
    from riffusion.riffusion_pipeline import DEFAULT_PARAMS, RiffusionPipeline
    from riffusion.spectrogram_params import SpectrogramParams
    from riffusion.text_to_audio_batch import parse_batch, plan_batch
    from riffusion.util.audio_util import AudioSegment

    calls = {}

    class FakePipe:
        def text_to_audio_batch(self, batch, **kw):
            calls.update(kw, batch=copy.deepcopy(batch))
            ps, entries = parse_batch(batch)
            clips, loops = plan_batch(ps, entries, kw["num_seeds"], kw["max_batch"])
            out = []
            for k, c in enumerate(clips):
                seg = AudioSegment(np.full((441 * (k + 1), 1), 100 * k, np.int16), 44100)
                out.append(dict(image=torch.full((512, 64, 3), k, dtype=torch.uint8), segment=seg))
            return dict(clips=out, loops=[dict(rows=list(lp.rows)) for lp in loops])

    monkeypatch.setattr(RiffusionPipeline, "load_checkpoint",
                        classmethod(lambda cls, checkpoint, device: calls.update(checkpoint=checkpoint) or FakePipe()))
    data = {"params": [{"name": "a", "guidance": 5.0}, {"name": "b", "checkpoint": "other/model"}],
            "entries": [{"prompt": "church bells", "seed": 3}, {"prompt": "jazz", "negative_prompt": "loud drums"}]}
    (tmp_path / "in.json").write_text(json.dumps(data))
    out_dir = tmp_path / "out"
    cli.main(["text-to-audio-batch", "--json", str(tmp_path / "in.json"), "--output-dir", str(out_dir),
              "--num-seeds", "2", "--max-batch", "3", "--checkpoint", "ckpt"])
    assert (calls["checkpoint"], calls["num_seeds"], calls["max_batch"], calls["batch"]) == ("ckpt", 2, 3, data)
    printed = capsys.readouterr().out
    assert "a: names checkpoint 'riffusion/riffusion-model-v1'" in printed and "b: names checkpoint 'other/model'" in printed
    names = [("church_bells_neg_", 3), ("church_bells_neg_", 4), ("jazz_neg_loud_drums", 42), ("jazz_neg_loud_drums", 43)]
    k = 0
    for stem, seed in names:
        for i in range(2):
            img = Image.open(out_dir / f"image_{i}_{stem}_{seed}.jpg")
            assert img.format == "JPEG" and img.size == (64, 512)
            assert SpectrogramParams.from_exif(img.getexif()) == DEFAULT_PARAMS
            seg = AudioSegment.from_file(str(out_dir / f"audio_{i}_{stem}_{seed}.wav"))
            assert abs(seg.duration_seconds - (k + 1) / 100) < 1e-9
            k += 1
    assert len(list(out_dir.iterdir())) == 2 * 8 + 1
    index = json.loads((out_dir / "index.json").read_text())
    assert [p["name"] for p in index["params"]] == ["a", "b"]
    e1 = index["entries"][1]
    assert [(o["name"], o["seed"]) for o in e1["outputs"]] == [("a", 42), ("b", 42), ("a", 43), ("b", 43)]
    assert e1["outputs"][-1]["audio_path"] == e1["audio_path"] == str(out_dir / "audio_1_jazz_neg_loud_drums_43.wav")
    assert all(Path(o["image_path"]).exists() for e in index["entries"] for o in e["outputs"])
    assert parse_batch(index) == parse_batch(data)
