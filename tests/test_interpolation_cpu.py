"""Interpolation without a GPU: the alphas, the per-row PLMS table of `PNDMRowsB200` against independent
`PNDMSchedulerB200` runs, the batched walk against per-request `riffuse` on a fake UNet, the evaluation counts, the
rejections, the operand contract of `cfg_pndm_rows_step`, the `interpolation` command and the bench script's accounting.
"""
import importlib.util
import sys
import types
from pathlib import Path

import numpy as np
import pytest
import torch
from PIL import Image

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "tests" / "golden"))


# ----------------------------------------------------------------------------------------------- alphas
@pytest.mark.parametrize("n", [1, 2, 5, 12, 20])
@pytest.mark.parametrize("p", [1.0, 2.0, 0.5])
def test_interpolation_alphas_are_the_pages(n, p):
    from riffusion.riffusion_pipeline import RiffusionPipeline

    alphas = np.linspace(0, 1, n)                           # streamlit/tasks/interpolation.py:99-104
    alphas_shifted = alphas * 2 - 1
    alphas_shifted = (np.abs(alphas_shifted) ** p * np.sign(alphas_shifted) + 1) / 2
    assert np.array_equal(RiffusionPipeline.interpolation_alphas(n, p), alphas_shifted)
    if n == 1:
        assert RiffusionPipeline.interpolation_alphas(n, p).tolist() == [0.0]


# ----------------------------------------------------------------------------------------------- the kernel's math
def _f32(v) -> float:
    """a coefficient as the kernel receives it: a C float"""
    return float(np.float32(v))


def _step_math(eu, et, g, coef, hist, base, ca, cb):
    """rf_cfg_pndm_step_f16 / rf_cfg_pndm_rows_step_f16 in the dtype of the tensors: guidance combine, then
    e = c0 eps + c1 h1 + c2 h2 + c3 h3 over the given terms, then prev = ca base - cb e"""
    eps = eu + _f32(g) * (et - eu)
    e = _f32(coef[0]) * eps
    for c, h in zip(coef[1:], hist):
        e = e + _f32(c) * h
    return eps, _f32(ca) * base - _f32(cb) * e


def _fake_pndm_step(eps_pair, guidance, hist, coef, sample, ca, cb, want_eps=True):
    n, d = sample.shape[0], torch.float64
    eps, prev = _step_math(eps_pair[:n].to(d), eps_pair[n:].to(d), guidance, coef, [h.to(d) for h in hist],
                           sample.to(d), ca, cb)
    return (eps.to(sample.dtype) if want_eps else None), prev.to(sample.dtype)


def _fake_rows_step(eps_pair, rows, ring, saved, sample):
    """the torch definition of rf_cfg_pndm_rows_step_f16, row by row"""
    from riffusion.scheduler_b200 import ROW_BASE_SAVED, ROW_DTYPE, ROW_SAVE

    B = sample.shape[0]
    table = rows.cpu().numpy().copy().view(ROW_DTYPE).reshape(B)
    prev = sample.clone()
    for r in range(B):
        rec = table[r]
        if not rec["active"]:
            continue
        slots = [int(rec[k]) for k in ("h1", "h2", "h3")]
        hist = [ring[s, r].to(torch.float64) for s in slots if 0 <= s < 4]
        coef = [float(rec["c0"])] + [float(rec[c]) for c, s in zip(("c1", "c2", "c3"), slots) if 0 <= s < 4]
        base = saved[r] if rec["flags"] & ROW_BASE_SAVED else sample[r]
        eps, p = _step_math(eps_pair[r].to(torch.float64), eps_pair[B + r].to(torch.float64), float(rec["guidance"]),
                            coef, hist, base.to(torch.float64), float(rec["ca"]), float(rec["cb"]))
        if 0 <= rec["push"] < 4:
            ring[int(rec["push"]), r] = eps.to(ring.dtype)
        if rec["flags"] & ROW_SAVE:
            saved[r] = sample[r]
        prev[r] = p.to(sample.dtype)
    return prev


@pytest.fixture
def fake_kernels(monkeypatch):
    from riffusion import scheduler_b200, tc_ops

    monkeypatch.setattr(tc_ops, "cfg_pndm_step", _fake_pndm_step)
    monkeypatch.setattr(scheduler_b200, "cfg_pndm_rows_step", _fake_rows_step)


# ----------------------------------------------------------------------------------------------- the row table
@pytest.mark.parametrize("steps", [50, 12])
def test_row_table_equals_independent_schedulers(fake_kernels, steps):
    """rows starting at 0, at 1 (the duplicated 961), in the middle, one step before the end and never, each with its
    own guidance: every row equals its own PNDMSchedulerB200 run over timesteps[t_start:], bit for bit (fp64)"""
    from riffusion.scheduler_b200 import PNDMRowsB200, PNDMSchedulerB200

    n_t = steps + 1
    t_starts = [0, 1, 2, steps // 2, n_t - 1, n_t, 1]
    guidances = [7.0, 5.5, 7.25, 9.0, 3.0, 7.0, 1.5]
    B = len(t_starts)
    rows = PNDMRowsB200(steps, t_starts, guidances, device="cpu")
    assert rows.t0 == 0 and len(rows.timesteps) == n_t
    assert (rows.table["active"].sum(axis=0) == [n_t - t for t in t_starts]).all()
    g = torch.Generator().manual_seed(5)
    x0 = torch.randn((B, 4, 3, 5), generator=g, dtype=torch.float64)
    pairs = [torch.randn((2 * B, 4, 3, 5), generator=g, dtype=torch.float64) for _ in range(n_t)]
    x = x0
    for j, t in enumerate(rows.timesteps):
        x = rows.step_cfg(pairs[j], 7.0, int(t), x)
    for r, (t_start, gr) in enumerate(zip(t_starts, guidances)):
        s = PNDMSchedulerB200()
        s.set_timesteps(steps)
        want = x0[r:r + 1]
        for i in range(t_start, n_t):
            pair = torch.cat([pairs[i][r:r + 1], pairs[i][B + r:B + r + 1]])
            want = s.step_cfg(pair, gr, int(s.timesteps[i]), want)
        assert torch.equal(x[r:r + 1], want), (r, t_start)
    with pytest.raises(ValueError, match="not timestep"):
        rows.step_cfg(pairs[0], 7.0, 1, x)


def test_row_table_records():
    """the records of a row started at 0: the first step saves its sample and pushes slot 0; the second restarts from
    the saved sample with one history term; pushes cycle through the 4 ring slots and never overwrite a slot read in the
    same step; no-guidance rows hold guidance 0; mixed sides and bad starts raise"""
    from riffusion.scheduler_b200 import ROW_BASE_SAVED, ROW_SAVE, PNDMRowsB200

    rows = PNDMRowsB200(10, [0, 4], [7.0, 8.0], device="cpu")
    t = rows.table
    assert t["flags"][0, 0] == ROW_SAVE and t["push"][0, 0] == 0 and t["h1"][0, 0] == -1
    assert t["flags"][1, 0] == ROW_BASE_SAVED and t["push"][1, 0] == -1 and t["h1"][1, 0] == 0
    assert (t["c0"][1, 0], t["c1"][1, 0]) == (0.5, 0.5)
    assert t["active"][:4, 1].tolist() == [0, 0, 0, 0] and t["flags"][4, 1] == ROW_SAVE
    for j in range(len(t)):
        for r in range(2):
            reads = {int(t[h][j, r]) for h in ("h1", "h2", "h3")} - {-1}
            assert int(t["push"][j, r]) not in reads
            assert reads <= {0, 1, 2, 3}
    assert t["guidance"][:, 0].max() == np.float32(7.0)
    assert np.all(PNDMRowsB200(10, [0, 3], [1.0, 0.5], device="cpu").table["guidance"] == 0)
    assert tuple(rows.rows.shape) == (11, 2, 13) and rows.rows.dtype == torch.int32
    with pytest.raises(ValueError, match="both sides of 1"):
        PNDMRowsB200(10, [0, 3], [7.0, 1.0], device="cpu")
    with pytest.raises(ValueError, match="t_starts must lie"):
        PNDMRowsB200(10, [0, 12], [7.0, 7.0], device="cpu")
    with pytest.raises(ValueError, match="one t_start and one guidance"):
        PNDMRowsB200(10, [0, 1], [7.0], device="cpu")


# ----------------------------------------------------------------------------------------------- the walk
class _FakeVae:
    """moments from an 8x average pool of the image; `config` as the pipeline reads it"""
    config = types.SimpleNamespace(block_out_channels=[1, 2, 3, 4])

    def encode_moments(self, img):
        pooled = torch.nn.functional.avg_pool2d(img.float(), 8)
        mean = torch.cat([pooled, pooled[:, :1]], dim=1)
        return mean.half(), (0.3 * mean - 1.5).half()


class _RowwiseUNet:
    """each row's output depends on that row only, so batch and single-request runs agree bit for bit"""

    def __init__(self):
        self.calls = []

    def __call__(self, x, t, encoder_hidden_states=None, **kw):
        self.calls.append((x.shape[0], int(t)))
        out = 0.3 * torch.tanh(x.float()) + 0.002 * (t / 1000.0) + \
            0.05 * encoder_hidden_states.float().mean(dim=(1, 2))[:, None, None, None]
        return types.SimpleNamespace(sample=out.to(torch.float16))


def _u8(scaled):
    return (scaled.float() * 40 + 128).clamp(0, 255).to(torch.uint8)[:, :3].permute(0, 2, 3, 1).contiguous()


@pytest.fixture
def walk_pipe(monkeypatch, fake_kernels):
    from prompt_stub import StubTextEncoder, StubTokenizer

    from riffusion import tc_ops
    from riffusion.riffusion_pipeline import RiffusionPipeline

    monkeypatch.setattr(tc_ops, "axpby", lambda x, noise, a, b, mask=None, z=None:
                        (a * x.float() + b * noise.float()).half())
    pipe = RiffusionPipeline(vae=_FakeVae(), unet=_RowwiseUNet(), text_encoder=StubTextEncoder(),
                             tokenizer=StubTokenizer(), device="cpu")
    pipe.use_cuda_graph = False
    pipe.device_slerp = False
    pipe._decode_u8 = _u8
    pipe._converter = lambda params, converter: None
    pipe._u8_to_waveform = lambda u8, conv, stereo, angles: \
        torch.sin(u8.float().mean(dim=(1, 3))[:, None, :].repeat(1, 1, 50) / 9.0)
    return pipe


def _image(seed=0, size=64):
    """a size x 512 seed image: 512 rows, as the default params' 512 frequencies need"""
    rng = np.random.default_rng(seed)
    return Image.fromarray(rng.integers(0, 256, (512, size, 3), dtype=np.uint8))


@pytest.mark.parametrize("den_a,den_b,max_batch", [(0.5, 0.9, 32), (0.75, 0.75, 32), (0.3, 0.8, 2)])
def test_walk_equals_riffuse_per_request(walk_pipe, den_a, den_b, max_batch):
    """every clip of the walk is `riffuse` of its request, bit for bit on a row-wise fake UNet with the torch definitions
    of the kernels; one loop per max_batch rows, each at the full batch"""
    from riffusion.datatypes import PromptInput

    pipe = walk_pipe
    a = PromptInput(prompt="church bells", seed=3, denoising=den_a, guidance=7.0)
    b = PromptInput(prompt="jazz (piano:1.2)", seed=8, denoising=den_b, guidance=5.0)
    img = _image()
    out = pipe.interpolation(a, b, img, num_interpolation_steps=5, num_inference_steps=10, max_batch=max_batch)
    assert len(out["n_unet_evals"]) == -(-5 // max_batch)
    assert out["alphas"].tolist() == [0.0, 0.25, 0.5, 0.75, 1.0]
    assert [r.alpha for r in out["requests"]] == out["alphas"].tolist()
    assert out["images"].shape == (5, 64, 8, 3) and out["waveform"].shape == (5, 1, 400)
    assert abs(out["segment"].duration_seconds - 5 * 400 / 44100) < 1e-9
    pipe.unet.calls.clear()
    for i, req in enumerate(out["requests"]):
        want = np.asarray(pipe.riffuse(req, img))
        assert np.array_equal(out["images"][i].numpy(), want), i


def test_walk_counts_on_the_page_defaults(walk_pipe):
    """12 alphas, 50 steps, guidance 7: ends at 0.75 run one loop of 38 evaluations (riffuse_batch: 2 groups); ends at
    0.5 / 0.9 one loop of 46 (riffuse_batch: 12 groups, 427 evaluations); every evaluation is at the full batch"""
    from riffusion.datatypes import PromptInput

    pipe = walk_pipe
    for den_a, den_b, want in ((0.75, 0.75, 38), (0.5, 0.9, 46)):
        pipe.unet.calls.clear()
        a = PromptInput(prompt="a", seed=1, denoising=den_a, guidance=7.0)
        b = PromptInput(prompt="b", seed=2, denoising=den_b, guidance=7.0)
        out = pipe.interpolation(a, b, _image(size=64))
        assert out["n_unet_evals"] == [want]
        assert pipe.unet.calls[0][0] == 24 and all(c[0] == 24 for c in pipe.unet.calls)


def test_rejections_before_any_unet_call(walk_pipe):
    from riffusion.datatypes import PromptInput

    pipe = walk_pipe
    a = PromptInput(prompt="a", seed=1, guidance=7.0)
    for kw, match in ((dict(num_interpolation_steps=0), "num_interpolation_steps"), (dict(max_batch=0), "max_batch")):
        with pytest.raises(ValueError, match=match):
            pipe.interpolation(a, a, _image(), **kw)
    with pytest.raises(ValueError, match="different sides of 1"):
        pipe.interpolation(a, PromptInput(prompt="b", seed=2, guidance=1.0), _image())
    with pytest.raises(ValueError, match="pixels high"):
        pipe.interpolation(a, a, _image().resize((64, 480)))
    assert not pipe.unet.calls


# ----------------------------------------------------------------------------------------------- operand contract
def _lat(*lead):
    return torch.zeros((*lead, 4, 8, 8), dtype=torch.float16)


def _rows(b):
    return torch.zeros((b, 13), dtype=torch.int32)


VALID = lambda: (_lat(4), _rows(2), _lat(4, 2), _lat(2), _lat(2))        # noqa: E731
MALFORMED = {
    "eps_pair_rows": lambda: (_lat(2), _rows(2), _lat(4, 2), _lat(2), _lat(2)),
    "eps_pair_dtype": lambda: (_lat(4).float(), _rows(2), _lat(4, 2), _lat(2), _lat(2)),
    "rows_count": lambda: (_lat(4), _rows(3), _lat(4, 2), _lat(2), _lat(2)),
    "rows_dtype": lambda: (_lat(4), _rows(2).float(), _lat(4, 2), _lat(2), _lat(2)),
    "rows_fields": lambda: (_lat(4), torch.zeros((2, 12), dtype=torch.int32), _lat(4, 2), _lat(2), _lat(2)),
    "ring_slots": lambda: (_lat(4), _rows(2), _lat(3, 2), _lat(2), _lat(2)),
    "ring_strided": lambda: (_lat(4), _rows(2), _lat(4, 4)[:, ::2], _lat(2), _lat(2)),
    "saved_shape": lambda: (_lat(4), _rows(2), _lat(4, 2), _lat(1), _lat(2)),
    "sample_empty": lambda: (_lat(0), _rows(0), _lat(4, 0), _lat(0), _lat(0)),
    "sample_dtype": lambda: (_lat(4), _rows(2), _lat(4, 2), _lat(2), _lat(2).float()),
}


@pytest.fixture
def recorder(monkeypatch):
    from riffusion import _native

    calls = []
    monkeypatch.setattr(_native, "is_device_tensor", lambda t: t.device.type == "cpu")
    monkeypatch.setattr(_native, "call", lambda name, device, *args: calls.append((name, args)))
    return calls


def test_rows_step_contract(recorder):
    from riffusion import _native
    from riffusion.scheduler_b200 import cfg_pndm_rows_step

    prev = cfg_pndm_rows_step(*VALID())
    assert [c[0] for c in recorder] == ["rf_cfg_pndm_rows_step_f16"] and recorder[0][1][1:3] == (2, 256)
    assert prev.shape == (2, 4, 8, 8) and prev.dtype == torch.float16
    for name, run in MALFORMED.items():
        recorder.clear()
        with pytest.raises((ValueError, _native.NativeError)):
            cfg_pndm_rows_step(*run())
        assert recorder == [], name


def test_rows_step_refuses_host_tensors(monkeypatch):
    from riffusion import _native
    from riffusion.scheduler_b200 import cfg_pndm_rows_step

    calls = []
    monkeypatch.setattr(_native, "call", lambda name, device, *args: calls.append(name))
    with pytest.raises(_native.NativeError, match="CUDA tensor"):
        cfg_pndm_rows_step(*VALID())
    assert calls == []


# ----------------------------------------------------------------------------------------------- CLI
def test_cli_interpolation_flags_and_defaults():
    from riffusion import cli

    sub = next(a for a in cli.build_parser()._actions if a.dest == "command")
    assert len(sub.choices) == 6 and "interpolation" not in sub.choices
    parser = cli.build_parser(cli.COMMANDS + cli.EXTRA_COMMANDS + cli.TRACK_COMMANDS)
    sub = next(a for a in parser._actions if a.dest == "command")
    flags = {o for act in sub.choices["interpolation"]._actions for o in act.option_strings}
    assert {"--prompt-a", "--prompt-b", "--seed-image", "--output", "--image-dir", "--seed-a", "--seed-b",
            "--denoising-a", "--denoising-b", "--guidance", "--num-interpolation-steps", "--num-inference-steps",
            "--alpha-power", "--max-batch", "--checkpoint", "--device"} <= flags
    with pytest.raises(SystemExit):
        parser.parse_args(["interpolation", "--prompt-a", "a", "--prompt-b", "b", "--output", "o.wav"])
    ns = parser.parse_args(["interpolation", "--prompt-a", "a", "--prompt-b", "b", "--seed-image", "s.png",
                            "--output", "o.wav"])
    assert (ns.seed_a, ns.seed_b, ns.denoising_a, ns.denoising_b, ns.guidance) == (42, 42, 0.75, 0.75, 7.0)
    assert (ns.num_interpolation_steps, ns.num_inference_steps, ns.alpha_power, ns.max_batch, ns.image_dir) == \
        (12, 50, 1.0, 32, "")


def test_cli_interpolation_writes_files(monkeypatch, tmp_path):
    from riffusion import cli
    from riffusion.riffusion_pipeline import DEFAULT_PARAMS, RiffusionPipeline
    from riffusion.util.audio_util import AudioSegment

    calls = {}

    class FakePipe:
        def interpolation(self, start, end, init_image, **kw):
            calls.update(kw, start=start, end=end, size=init_image.size)
            seg = AudioSegment(np.zeros((44100 * 3, 1), np.int16), 44100)
            return dict(segment=seg, images=torch.full((3, 64, 80, 3), 9, dtype=torch.uint8), alphas=np.zeros(3))

    monkeypatch.setattr(RiffusionPipeline, "load_checkpoint",
                        classmethod(lambda cls, checkpoint, device: calls.update(checkpoint=checkpoint) or FakePipe()))
    _image(size=96).save(tmp_path / "seed.png")
    cli.main(["interpolation", "--prompt-a", "jazz", "--prompt-b", "rock", "--seed-image", str(tmp_path / "seed.png"),
              "--output", str(tmp_path / "out.wav"), "--image-dir", str(tmp_path / "img"), "--denoising-b", "0.9",
              "--seed-b", "7", "--num-interpolation-steps", "3", "--checkpoint", "ckpt"])
    assert (calls["start"].prompt, calls["start"].seed, calls["start"].denoising, calls["start"].guidance) == \
        ("jazz", 42, 0.75, 7.0)
    assert (calls["end"].prompt, calls["end"].seed, calls["end"].denoising) == ("rock", 7, 0.9)
    assert (calls["num_interpolation_steps"], calls["num_inference_steps"], calls["alpha_power"], calls["max_batch"],
            calls["checkpoint"], calls["size"]) == (3, 50, 1.0, 32, "ckpt", (96, 512))
    assert abs(AudioSegment.from_file(str(tmp_path / "out.wav")).duration_seconds - 3.0) < 1e-9
    from riffusion.spectrogram_params import SpectrogramParams

    for i in range(3):
        img = Image.open(tmp_path / "img" / f"step_{i}.png")
        assert img.size == (80, 64) and np.asarray(img)[0, 0, 0] == 9
        assert SpectrogramParams.from_exif(img.getexif()) == DEFAULT_PARAMS


# ----------------------------------------------------------------------------------------------- bench
def test_bench_script_accounting():
    spec = importlib.util.spec_from_file_location("bench_interpolation", ROOT / "tools" / "bench_interpolation.py")
    mod = importlib.util.module_from_spec(spec)
    sys.modules["bench_interpolation"] = mod
    spec.loader.exec_module(mod)
    same = mod.walk_accounting(12, 50, 0.75, 0.75, 32)
    assert same["rows"] == {"loops": 1, "unet_evals": 38, "cfg_batch": 24, "row_evals": 456, "idle_row_evals": 0}
    assert same["grouped"] == {"loops": 2, "unet_evals": 76}
    diff = mod.walk_accounting(12, 50, 0.5, 0.9, 32)
    assert diff["rows"] == {"loops": 1, "unet_evals": 46, "cfg_batch": 24, "row_evals": 552, "idle_row_evals": 125}
    assert diff["grouped"] == {"loops": 12, "unet_evals": 427}
    assert mod.walk_accounting(12, 50, 0.5, 0.9, 5)["rows"]["loops"] == 3
