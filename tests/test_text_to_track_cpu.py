"""Long tracks without a GPU: the canvas geometry, the overlap weights, prompt spans -> windows, loop grouping, the
refusals (all before any device work), the operand contracts of `window_ops` and the `text-to-track` command."""
from __future__ import annotations

import numpy as np
import pytest
import torch

F16, F32 = torch.float16, torch.float32


# ------------------------------------------------------------------------------------- geometry and weights
@pytest.mark.parametrize("duration,frames,width,n", [(30.0, 3001, 3072, 11), (60.0, 6001, 6144, 23),
                                                     (120.0, 12001, 12032, 46), (5.0, 501, 512, 1),
                                                     (5.12, 513, 768, 2), (0.01, 2, 512, 1)])
def test_track_geometry(duration, frames, width, n):
    from riffusion.riffusion_pipeline import RiffusionPipeline

    assert RiffusionPipeline.track_geometry(duration, 512, 256, 441, 44100) == (frames, width, n)


def test_canvas_width_other_strides():
    from riffusion import window_ops

    assert window_ops.canvas_width(3001, 512, 512) == 3072
    assert window_ops.canvas_width(3001, 512, 128) == 3072
    assert window_ops.canvas_width(3001, 256, 64) == 3008
    assert window_ops.window_count(3008, 256, 64) == 44


@pytest.mark.parametrize("Ww,s,n", [(64, 32, 5), (64, 16, 6), (64, 8, 9), (64, 64, 4), (64, 48, 3), (64, 32, 1),
                                    (32, 24, 2)])
def test_merge_weights_sum_to_one(Ww, s, n):
    from riffusion import window_ops

    wn = window_ops.merge_weights(Ww, s, n)
    assert wn.shape == (n, Ww) and wn.dtype == np.float32
    total = np.zeros(Ww + (n - 1) * s)
    cover = np.zeros_like(total)
    for k in range(n):
        total[k * s:k * s + Ww] += wn[k]
        cover[k * s:k * s + Ww] += 1
    assert np.abs(total - 1).max() < 1e-6
    assert np.all(wn > 0)
    # a column one window covers alone has weight exactly 1
    for k in range(n):
        alone = cover[k * s:k * s + Ww] == 1
        assert np.all(wn[k][alone] == 1.0)


def test_raw_weights_are_linear_ramps_at_half_stride():
    from riffusion import window_ops

    Ww, s, n = 64, 32, 4
    w = window_ops.raw_weights(Ww, s, n)
    c = np.arange(Ww) + 0.5
    up, down = np.minimum(1, c / 32), np.minimum(1, (Ww - c) / 32)
    assert np.array_equal(w[0], down) and np.array_equal(w[n - 1], up)
    assert np.array_equal(w[1], np.minimum(up, down))
    wn = window_ops.merge_weights(Ww, s, n)
    # neighbours crossfade linearly over the overlap: window k's second half and window k+1's first half sum to 1
    assert np.allclose(wn[1, 32:], (Ww - c[32:]) / 32) and np.allclose(wn[2, :32], c[:32] / 32)
    assert np.allclose(wn[1, 32:] + wn[2, :32], 1.0)


def test_weights_without_overlap_are_one():
    from riffusion import window_ops

    assert np.array_equal(window_ops.raw_weights(64, 64, 3), np.ones((3, 64)))
    assert np.array_equal(window_ops.merge_weights(64, 64, 3), np.ones((3, 64), dtype=np.float32))


@pytest.mark.parametrize("width,Ww,s,message", [(1000, 512, 256, "multiple of 64"), (768, 512, 0, "multiple of 64"),
                                                (768, 512, 640, "exceeds"), (832, 512, 256, "whole number"),
                                                (256, 512, 256, "whole number"), (768, 500, 256, "multiple of 64")])
def test_window_count_refusals(width, Ww, s, message):
    from riffusion import window_ops

    with pytest.raises(ValueError, match=message):
        window_ops.window_count(width, Ww, s)


# ------------------------------------------------------------------------------------- prompts and loops
def test_prompt_spans_to_windows():
    from riffusion.riffusion_pipeline import RiffusionPipeline

    pick = RiffusionPipeline.track_prompts
    assert pick("piano", 3, 512, 256, 441, 44100) == ["piano"] * 3
    # window centres at 2.56, 5.12, 7.68, 10.24 s
    spans = [(0, "a"), (5.12, "b"), (9, "c")]
    assert pick(spans, 4, 512, 256, 441, 44100) == ["a", "b", "b", "c"]
    assert pick([(0, "a"), (100, "b")], 4, 512, 256, 441, 44100) == ["a"] * 4


@pytest.mark.parametrize("spans,message", [([], "no prompt spans"), ([(1, "a")], "start at 0"),
                                           ([(0, "a"), (5, "b"), (5, "c")], "strictly increase"),
                                           ([(0, "a"), (5, "b"), (3, "c")], "strictly increase")])
def test_prompt_span_refusals(spans, message):
    from riffusion.riffusion_pipeline import RiffusionPipeline

    with pytest.raises(ValueError, match=message):
        RiffusionPipeline.track_prompts(spans, 3, 512, 256, 441, 44100)


@pytest.mark.parametrize("tracks,n,max_batch,loops", [(4, 23, 32, [[0], [1], [2], [3]]), (4, 11, 32, [[0, 1], [2, 3]]),
                                                      (3, 11, 22, [[0, 1], [2]]), (5, 1, 2, [[0, 1], [2, 3], [4]]),
                                                      (1, 46, 32, [[0]]), (2, 8, 64, [[0, 1]])])
def test_track_loops(tracks, n, max_batch, loops):
    from riffusion.riffusion_pipeline import RiffusionPipeline

    assert RiffusionPipeline.track_loops(tracks, n, max_batch) == loops


# ------------------------------------------------------------------------------------- refusals before device work
@pytest.fixture
def hostile_pipe(monkeypatch):
    """a pipeline whose every device-touching step fails loudly: a refusal must come first"""
    from riffusion import _native
    from riffusion.riffusion_pipeline import RiffusionPipeline

    def device_work(*a, **k):
        raise AssertionError("device work before the refusal")

    monkeypatch.setattr(_native, "call", device_work)
    pipe = RiffusionPipeline(vae=None, unet=None, device="cuda")
    for name in ("_converter", "embed_text", "_context", "_denoise", "_finish"):
        monkeypatch.setattr(pipe, name, device_work)
    monkeypatch.setattr(torch, "Generator", device_work)
    return pipe


@pytest.mark.parametrize("kw,message", [
    (dict(duration_s=0.0), "duration_s"), (dict(duration_s=121.0), "duration_s"), (dict(duration_s=-3.0), "duration_s"),
    (dict(stride=0), "stride"), (dict(stride=1024), "exceeds"), (dict(window_width=500), "window_width"),
    (dict(prompt=[]), "no prompt spans"), (dict(prompt=[(2.0, "a")]), "start at 0"),
    (dict(prompt=[(0, "a"), (0, "b")]), "strictly increase"), (dict(scheduler="LMSDiscreteScheduler"), "unsupported"),
    (dict(scheduler="EulerDiscreteScheduler"), "unsupported"), (dict(num_tracks=0), "num_tracks"),
    (dict(max_batch=0), "max_batch")])
def test_text_to_track_refuses_before_device_work(hostile_pipe, kw, message):
    kw = dict(kw)
    prompt = kw.pop("prompt", "piano")
    with pytest.raises(ValueError, match=message):
        hostile_pipe.text_to_track(prompt, **kw)


@pytest.mark.parametrize("kw,message", [
    (dict(width=1000), "multiple of 64"), (dict(width=832), "whole number"), (dict(height=100), "height"),
    (dict(prompt=["a", "b"]), "2 prompts for 3 windows"), (dict(num_tracks=0), "num_tracks"),
    (dict(max_batch=0), "max_batch"), (dict(scheduler="LMSDiscreteScheduler"), "unsupported")])
def test_txt2img_track_refuses_before_device_work(hostile_pipe, kw, message):
    kw = dict(kw)
    prompt = kw.pop("prompt", "piano")
    kw.setdefault("width", 1024)
    with pytest.raises(ValueError, match=message):
        hostile_pipe.txt2img_track(prompt, **kw)


# ------------------------------------------------------------------------------------- operand contracts
class _SizeQueries:
    pass


@pytest.fixture
def recorder(monkeypatch):
    from riffusion import _native

    calls = []
    monkeypatch.setattr(_native, "is_device_tensor", lambda t: t.device.type in ("cpu", "meta"))
    monkeypatch.setattr(_native, "call", lambda name, device, *args: calls.append((name, args)))
    monkeypatch.setattr(_native, "lib", lambda: _SizeQueries)
    return calls


def _win(Ww=8, s=8, n=3, dtype=F32, device="cpu"):
    from riffusion import window_ops

    return window_ops.Windows(Ww, s, n, torch.zeros((n, Ww), dtype=dtype, device=device))


def h(*shape, dtype=F16, device="cpu"):
    return torch.zeros(shape, dtype=dtype, device=device)


def test_window_ops_well_formed_calls(recorder):
    from riffusion import window_ops

    win = _win(16, 8, 3)
    out = window_ops.window_gather(h(4, 4, 2, 32), win)
    assert out.shape == (12, 4, 2, 16)
    merged = window_ops.window_merge(h(12, 4, 2, 16), win)
    assert merged.shape == (4, 4, 2, 32)
    assert [name for name, _ in recorder] == ["rf_window_gather_f16", "rf_window_merge_f16"]
    assert recorder[0][1][1:8] == (4, 4, 2, 32, 16, 8, 3)
    assert recorder[1][1][2:9] == (4, 4, 2, 32, 16, 8, 3)


@pytest.mark.parametrize("name,expected,run", [
    ("gather_canvas_width", ValueError, lambda wo: wo.window_gather(h(2, 4, 2, 40), _win(16, 8, 3))),
    ("gather_dtype", "NativeError", lambda wo: wo.window_gather(h(2, 4, 2, 32, dtype=F32), _win(16, 8, 3))),
    ("gather_dims", ValueError, lambda wo: wo.window_gather(h(4, 2, 32), _win(16, 8, 3))),
    ("gather_strided", ValueError, lambda wo: wo.window_gather(h(2, 4, 2, 64)[..., ::2], _win(16, 8, 3))),
    ("merge_width", ValueError, lambda wo: wo.window_merge(h(6, 4, 2, 24), _win(16, 8, 3))),
    ("merge_groups", ValueError, lambda wo: wo.window_merge(h(7, 4, 2, 16), _win(16, 8, 3))),
    ("merge_dtype", "NativeError", lambda wo: wo.window_merge(h(6, 4, 2, 16, dtype=F32), _win(16, 8, 3))),
    ("merge_strided", ValueError, lambda wo: wo.window_merge(h(6, 4, 16, 2).transpose(2, 3), _win(16, 8, 3))),
    ("merge_weights_dtype", "NativeError", lambda wo: wo.window_merge(h(6, 4, 2, 16), _win(16, 8, 3, dtype=F16))),
    ("merge_weights_shape", ValueError, lambda wo: wo.window_merge(
        h(6, 4, 2, 16), wo.Windows(16, 8, 3, torch.zeros(2, 16)))),
    ("merge_weights_device", ValueError, lambda wo: wo.window_merge(h(6, 4, 2, 16), _win(16, 8, 3, device="meta"))),
])
def test_window_ops_malformed_operands_raise_before_the_call(recorder, name, expected, run):
    from riffusion import _native, window_ops

    with pytest.raises(_native.NativeError if expected == "NativeError" else expected):
        run(window_ops)
    assert recorder == []


def test_window_ops_refuse_host_tensors(monkeypatch):
    from riffusion import _native, window_ops

    calls = []
    monkeypatch.setattr(_native, "call", lambda name, device, *args: calls.append(name))
    with pytest.raises(_native.NativeError, match="CUDA tensor"):
        window_ops.window_gather(h(2, 4, 2, 32), _win(16, 8, 3))
    with pytest.raises(_native.NativeError, match="CUDA tensor"):
        window_ops.window_merge(h(6, 4, 2, 16), _win(16, 8, 3))
    assert calls == []


def test_window_entry_points_are_declared():
    from pathlib import Path

    from riffusion import _native

    header = (Path(__file__).resolve().parents[1] / "include" / "rf_b200.h").read_text()
    for name in ("rf_window_gather_f16", "rf_window_merge_f16"):
        assert name in _native.SIGNATURES and f"int {name}(" in header


# ------------------------------------------------------------------------------------- command line
def test_parse_prompt_changes():
    from riffusion import cli

    assert cli.parse_prompt_changes("piano", "") == "piano"
    assert cli.parse_prompt_changes("piano", "20:jazz with drums;40:hard rock") == [
        (0.0, "piano"), (20.0, "jazz with drums"), (40.0, "hard rock")]
    assert cli.parse_prompt_changes("piano", "7.5: strings ") == [(0.0, "piano"), (7.5, "strings")]
    for bad in ("jazz", "x:jazz", "20:", "20:jazz;", ":jazz"):
        with pytest.raises(ValueError, match="prompt-changes"):
            cli.parse_prompt_changes("piano", bad)


def test_text_to_track_command_flags_and_defaults(monkeypatch, tmp_path):
    from riffusion import cli
    from riffusion.riffusion_pipeline import RiffusionPipeline

    assert cli.TRACK_COMMANDS[-1] is cli.text_to_track
    parser = cli.build_parser(cli.COMMANDS + cli.EXTRA_COMMANDS + cli.TRACK_COMMANDS)
    args = vars(parser.parse_args(["text-to-track", "--prompt", "piano", "--audio", "o.wav"]))
    args.pop("_fn"), args.pop("command")
    assert args == dict(prompt="piano", audio="o.wav", image="", prompt_changes="", negative_prompt="", duration_s=30.0,
                        seed=42, num_tracks=1, num_inference_steps=30, guidance=7.0,
                        scheduler="DPMSolverMultistepScheduler", window_width=512, stride=256, max_batch=32,
                        use_20k=False, checkpoint="riffusion/riffusion-model-v1", device="cuda")

    seen = {}

    class FakePipe:
        def text_to_track(self, prompt, **kw):
            seen.update(kw, prompt=prompt)
            T_ = kw["num_tracks"]
            L = round(kw["duration_s"] * 44100)
            return dict(images=torch.zeros(T_, 512, 768, 3, dtype=torch.uint8),
                        waveform=torch.sin(torch.arange(L, dtype=torch.float32) / 7).expand(T_, 1, L) * 1000,
                        windows=[dict(offset=0, prompt=prompt), dict(offset=256, prompt=prompt)])

    monkeypatch.setattr(RiffusionPipeline, "load_checkpoint", classmethod(lambda cls, **kw: FakePipe()))
    cli.main(["text-to-track", "--prompt", "piano", "--prompt-changes", "3:rock", "--audio", str(tmp_path / "t.wav"),
              "--image", str(tmp_path / "t.png"), "--duration-s", "6", "--num-tracks", "2", "--seed", "5",
              "--stride", "128", "--window-width", "256", "--max-batch", "8", "--guidance", "5",
              "--scheduler", "DDIMScheduler", "--negative-prompt", "noise"])
    assert seen["prompt"] == [(0.0, "piano"), (3.0, "rock")]
    assert (seen["duration_s"], seen["stride"], seen["window_width"], seen["max_batch"]) == (6.0, 128, 256, 8)
    assert (seen["guidance_scale"], seen["scheduler"], seen["negative_prompt"], seen["seed"]) == (5.0, "DDIMScheduler",
                                                                                                   "noise", 5)
    for s in (5, 6):
        assert (tmp_path / f"t_{s}.wav").exists() and (tmp_path / f"t_{s}.png").exists()


def test_text_to_track_command_refuses_before_loading(monkeypatch, tmp_path):
    from riffusion import cli
    from riffusion.riffusion_pipeline import RiffusionPipeline

    def load(cls, **kw):
        raise AssertionError("loaded the checkpoint before refusing")

    monkeypatch.setattr(RiffusionPipeline, "load_checkpoint", classmethod(load))
    for argv, message in ((["--duration-s", "200"], "duration_s"), (["--stride", "100"], "stride"),
                          (["--prompt-changes", "0:rock"], "strictly increase"),
                          (["--prompt-changes", "rock"], "prompt-changes")):
        with pytest.raises(ValueError, match=message):
            cli.main(["text-to-track", "--prompt", "piano", "--audio", str(tmp_path / "x.wav")] + argv)
