"""The batched model server without a GPU: the masked row table of `PNDMRowsB200` against per-row schedulers plus the
inpainting blend, `riffuse_requests` against per-request `riffuse` on a row-wise fake UNet with the torch definitions of
the kernels, the loop plan (groups, power-of-two batches, filler rows), `compute_requests`' responses and refusals,
`InferenceBatcher`'s batching and shutdown, the operand contract of `cfg_pndm_rows_mask_step` and the bench script's
accounting."""
import importlib.util
import json
import sys
import threading
import time
from pathlib import Path

import numpy as np
import pytest
import torch
from PIL import Image

from test_interpolation_cpu import _FakeVae, _fake_pndm_step, _fake_rows_step, _RowwiseUNet, _u8

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "tests" / "golden"))


def _fake_axpby(x, noise, a, b, mask=None, z=None):
    """the torch definition of rf_axpby_f16 in fp32, rounded once"""
    v = a * x.float() + b * noise.float()
    if mask is not None:
        m = mask.float()
        v = v * m + z.float() * (1 - m)
    return v.to(x.dtype)


def _fake_rows_mask_step(eps_pair, rows, ring, saved, sample, init, noise, mask, a, b):
    """the torch definition of rf_cfg_pndm_rows_mask_step_f16: the rows step, then rf_axpby_f16's blend on the rows
    whose record holds ROW_MASK (and only those read init / noise / mask)"""
    from riffusion.scheduler_b200 import ROW_DTYPE, ROW_MASK

    prev = _fake_rows_step(eps_pair, rows, ring, saved, sample)
    table = rows.cpu().numpy().copy().view(ROW_DTYPE).reshape(sample.shape[0])
    for r, rec in enumerate(table):
        if rec["active"] and rec["flags"] & ROW_MASK:
            prev[r] = _fake_axpby(init[r], noise[r], a, b, mask[r], prev[r])
    return prev


@pytest.fixture
def fake_kernels(monkeypatch):
    from riffusion import scheduler_b200, tc_ops

    monkeypatch.setattr(tc_ops, "cfg_pndm_step", _fake_pndm_step)
    monkeypatch.setattr(tc_ops, "axpby", _fake_axpby)
    monkeypatch.setattr(scheduler_b200, "cfg_pndm_rows_step", _fake_rows_step)
    monkeypatch.setattr(scheduler_b200, "cfg_pndm_rows_mask_step", _fake_rows_mask_step)


# ----------------------------------------------------------------------------------------------- the row table
@pytest.mark.parametrize("sched_name", ["PNDMScheduler", "DDIMScheduler"])
def test_masked_rows_equal_schedulers_plus_blend(fake_kernels, sched_name):
    """rows with and without a mask, starting at different steps: every row equals its own scheduler run followed,
    when masked, by add_noise(init, noise, t, mask, blend_with) at each of its steps, bit for bit (fp64); the unmasked
    and not yet started rows never read their NaN blend inputs"""
    from riffusion.scheduler_b200 import SCHEDULERS, PNDMRowsB200

    cls = SCHEDULERS[sched_name]
    steps = 12
    probe = cls()
    probe.set_timesteps(steps)
    n_t = len(probe.timesteps)
    t_starts = [0, 1, 5, n_t - 1, n_t, 3]
    guidances = [7.0, 5.5, 9.0, 6.0, 7.0, 8.25]
    masked = [True, False, True, True, False, False]
    B = len(t_starts)
    rows = PNDMRowsB200(steps, t_starts, guidances, device="cpu", scheduler=cls, masked=masked)
    g = torch.Generator().manual_seed(3)
    shape = (B, 4, 3, 5)
    x0 = torch.randn(shape, generator=g, dtype=torch.float64)
    init = torch.randn(shape, generator=g, dtype=torch.float64)
    noise = torch.randn(shape, generator=g, dtype=torch.float64)
    mask = (torch.rand(shape, generator=g) > 0.5).double()
    for r in range(B):
        if not masked[r]:
            init[r], noise[r], mask[r] = float("nan"), float("nan"), float("nan")
    rows.set_mask_inputs(init=init, noise=noise, mask=mask)
    pairs = [torch.randn((2 * B,) + shape[1:], generator=g, dtype=torch.float64) for _ in range(n_t)]
    x = x0
    for j, t in enumerate(rows.timesteps):
        x = rows.step_cfg(pairs[j], 7.0, int(t), x)
    for r in range(B):
        s = cls()
        s.set_timesteps(steps)
        want = x0[r:r + 1]
        for i in range(t_starts[r], n_t):
            t = int(s.timesteps[i])
            pair = torch.cat([pairs[i][r:r + 1], pairs[i][B + r:B + r + 1]])
            want = s.step_cfg(pair, guidances[r], t, want)
            if masked[r]:
                want = s.add_noise(init[r:r + 1], noise[r:r + 1], t, mask=mask[r:r + 1], blend_with=want)
        assert torch.equal(x[r:r + 1], want), r
    assert not torch.isnan(x).any()


def test_unmasked_table_is_unchanged():
    """no masks (None or all False): the table is byte for byte the plain one and the plain kernel runs; a mask only
    adds ROW_MASK to the masked rows' active steps"""
    from riffusion.scheduler_b200 import ROW_MASK, PNDMRowsB200

    args = (20, [0, 4, 21, 9], [7.0, 5.0, 6.0, 9.0])
    plain = PNDMRowsB200(*args, device="cpu")
    assert plain.table.tobytes() == PNDMRowsB200(*args, device="cpu", masked=[False] * 4).table.tobytes()
    assert not (plain.table["flags"] & ROW_MASK).any() and not plain.masked
    m = PNDMRowsB200(*args, device="cpu", masked=[True, False, True, True])
    want = plain.table.copy()
    want["flags"][:, [0, 2, 3]] |= ROW_MASK * want["active"][:, [0, 2, 3]]
    assert m.table.tobytes() == want.tobytes()
    assert torch.equal(m.rows, torch.from_numpy(want.view(np.int32).reshape(m.rows.shape)))
    with pytest.raises(ValueError, match="set_mask_inputs"):
        m.step_cfg(torch.zeros((8, 4, 2, 2)), 7.0, int(m.timesteps[0]), torch.zeros((4, 4, 2, 2)))
    with pytest.raises(ValueError, match="no row of this table is masked"):
        plain.set_mask_inputs(init=None, noise=None, mask=None)
    with pytest.raises(ValueError, match="one masked flag per row"):
        PNDMRowsB200(*args, device="cpu", masked=[True])


def test_plain_table_launches_the_plain_kernel(monkeypatch):
    from riffusion import scheduler_b200
    from riffusion.scheduler_b200 import PNDMRowsB200

    calls = []
    monkeypatch.setattr(scheduler_b200, "cfg_pndm_rows_step", lambda *a: calls.append("plain") or a[4])
    monkeypatch.setattr(scheduler_b200, "cfg_pndm_rows_mask_step", lambda *a: calls.append("mask") or a[4])
    x = torch.zeros((2, 4, 2, 2))
    for masked, kind in ((None, "plain"), ([False, True], "mask")):
        calls.clear()
        rows = PNDMRowsB200(5, [0, 2], [7.0, 7.0], device="cpu", masked=masked)
        if rows.masked:
            rows.set_mask_inputs(init=x, noise=x, mask=x)
        for t in rows.timesteps:
            rows.step_cfg(torch.zeros((4, 4, 2, 2)), 7.0, int(t), x)
        assert calls == [kind] * len(rows.timesteps)


# ----------------------------------------------------------------------------------------------- riffuse_requests
@pytest.fixture
def req_pipe(fake_kernels):
    from prompt_stub import StubTextEncoder, StubTokenizer

    from riffusion.riffusion_pipeline import RiffusionPipeline

    pipe = RiffusionPipeline(vae=_FakeVae(), unet=_RowwiseUNet(), text_encoder=StubTextEncoder(),
                             tokenizer=StubTokenizer(), device="cpu")
    pipe.use_cuda_graph = False
    pipe.device_slerp = False
    pipe._decode_u8 = _u8
    pipe._converter = lambda params, converter: None
    pipe._u8_to_waveform = lambda u8, conv, stereo, angles: \
        torch.sin(u8.float().mean(dim=(1, 3))[:, None, :].repeat(1, 1, 50) / 9.0) + \
        (0 if angles is None else angles.real.mean(dim=(1, 2, 3))[:, None, None])
    return pipe


def _image(seed=0, width=64):
    rng = np.random.default_rng(seed)
    return Image.fromarray(rng.integers(0, 256, (512, width, 3), dtype=np.uint8))


def _mask(width=64):
    m = np.zeros((512, width, 3), np.uint8)
    m[:, width // 2:] = 255
    return Image.fromarray(m)


LONG_PROMPT = " ".join(f"word{i}" for i in range(90))        # 92 tokens: a 154-token weighted context


def _mixed_requests():
    """mixed alphas, denoising 0.5 .. 0.9, guidance 5 .. 9, two seed images (two widths), masked and unmasked rows, two
    context lengths.  The 154-token prompts run without guidance: with it, riffuse (as the reference) cannot join
    their context to the 77-token unconditional one."""
    from riffusion.datatypes import InferenceInput, PromptInput

    reqs, images, masks = [], [], []
    specs = [(0.0, 0.5, 0.9, 5.0, 9.0, 0, True, False), (0.25, 0.75, 0.75, 7.0, 7.0, 0, False, False),
             (0.5, 0.6, 0.8, 6.0, 8.0, 1, True, False), (1.0, 0.5, 0.9, 9.0, 5.0, 1, False, False),
             (0.75, 0.9, 0.5, 1.0, 0.5, 0, True, True), (0.3, 0.75, 0.75, 0.9, 0.6, 0, False, True),
             (0.6, 0.7, 0.9, 7.0, 7.0, 0, False, False), (0.1, 0.55, 0.85, 5.5, 8.5, 1, True, False),
             (0.4, 0.6, 0.8, 1.0, 1.0, 0, True, False)]
    for k, (alpha, d0, d1, g0, g1, img, masked, long_ctx) in enumerate(specs):
        start = PromptInput(prompt=LONG_PROMPT if long_ctx else "church bells", seed=3 + k, denoising=d0, guidance=g0)
        end = PromptInput(prompt="jazz (piano:1.2)", seed=40 + k, denoising=d1, guidance=g1)
        if long_ctx:
            end = PromptInput(prompt=LONG_PROMPT + " drums", seed=40 + k, denoising=d1, guidance=g1)
        reqs.append(InferenceInput(alpha=alpha, num_inference_steps=10, start=start, end=end))
        width = 64 if img == 0 else 96
        images.append(_image(img, width))
        masks.append(_mask(width) if masked else None)
    return reqs, images, masks


@pytest.mark.parametrize("max_batch", [1, 3, 16])
def test_riffuse_requests_equal_riffuse(req_pipe, max_batch):
    """every request's image is `riffuse` of it, bit for bit on a row-wise fake UNet, at every max_batch"""
    pipe = req_pipe
    reqs, images, masks = _mixed_requests()
    assert pipe.embed_text_weighted(LONG_PROMPT).shape[1] == 154
    outs = pipe.riffuse_requests(reqs, images, masks, max_batch=max_batch)
    assert len(outs) == len(reqs)
    for i, (req, img, mask) in enumerate(zip(reqs, images, masks)):
        want = np.asarray(pipe.riffuse(req, img, mask_image=mask))
        assert np.array_equal(outs[i]["image"].numpy(), want), i
    loops = {o["loop"] for o in outs}
    assert len(loops) == len(pipe.request_loops(_keys(pipe, reqs, images), max_batch))


def _keys(pipe, reqs, images):
    return [(r.num_inference_steps, (im.height // 8, im.width // 8), pipe.embed_text_weighted(r.start.prompt).shape[1],
             (r.start.guidance * (1 - r.alpha) + r.end.guidance * r.alpha) > 1.0) for r, im in zip(reqs, images)]


def test_request_loops_groups_and_buckets():
    from riffusion.riffusion_pipeline import RiffusionPipeline

    keys = ["a"] * 11 + ["b"] * 3 + ["a", "c"]
    loops = RiffusionPipeline.request_loops(keys, 8)
    assert [(len(i), b) for i, b in loops] == [(8, 8), (4, 4), (3, 4), (1, 1)]
    assert loops[0][0] == list(range(8)) and loops[1][0] == [8, 9, 10, 14] and loops[2][0] == [11, 12, 13]
    assert [b for _, b in RiffusionPipeline.request_loops(["k"] * 5, 16)] == [8]
    assert [b for _, b in RiffusionPipeline.request_loops(["k"] * 5, 6)] == [6]
    assert [b for _, b in RiffusionPipeline.request_loops(["k"] * 3, 3)] == [3]
    assert [b for _, b in RiffusionPipeline.request_loops(["k"] * 17, 16)] == [16, 1]
    for n in range(1, 40):
        for mb in (1, 2, 3, 5, 16):
            for idx, b in RiffusionPipeline.request_loops(["k"] * n, mb):
                assert len(idx) <= b <= mb and (b == mb or b & (b - 1) == 0) and b < 2 * len(idx)
    with pytest.raises(ValueError, match="max_batch"):
        RiffusionPipeline.request_loops(["k"], 0)


def test_filler_rows_never_step_and_are_dropped(req_pipe):
    """5 compatible requests run as one loop of 8 rows: the UNet sees the batch of 8, the 3 filler rows report
    themselves and produce no output; the real rows are still riffuse's"""
    pipe = req_pipe
    reqs, _, _ = _mixed_requests()
    reqs = [reqs[i] for i in (0, 1, 6, 0, 1)]          # one group: one seed image, 77-token prompts, guidance above 1
    images, masks = [_image(0)] * 5, [None, _mask(), None, _mask(), None]
    pipe.unet.calls.clear()
    outs = pipe.riffuse_requests(reqs, images, masks, max_batch=16)
    assert len(outs) == 5 and {o["loop"] for o in outs} == {0} and {o["filler_rows"] for o in outs} == {3}
    assert all(c[0] == 16 for c in pipe.unet.calls) and len(pipe.unet.calls) == outs[0]["n_unet_evals"]
    for o, req, img, mask in zip(outs, reqs, images, masks):
        assert np.array_equal(o["image"].numpy(), np.asarray(pipe.riffuse(req, img, mask_image=mask)))


def test_filler_rows_table(monkeypatch, req_pipe):
    """the filler rows of a loop are never active"""
    from riffusion import scheduler_b200

    made = []
    real = scheduler_b200.PNDMRowsB200

    class Spy(real):
        def __init__(self, *a, **kw):
            super().__init__(*a, **kw)
            made.append(self)

    monkeypatch.setattr(scheduler_b200, "PNDMRowsB200", Spy)
    reqs, images, masks = _mixed_requests()
    req_pipe.riffuse_requests(reqs[:3], [images[0]] * 3, [None] * 3, max_batch=16)
    assert len(made) == 1 and made[0].table.shape[1] == 4
    assert not made[0].table["active"][:, 3].any() and made[0].table["active"][:, :3].any(axis=0).all()


def test_riffuse_requests_refusals(req_pipe):
    from riffusion.scheduler_b200 import DPMSolverMultistepSchedulerB200, EulerAncestralSchedulerB200

    pipe = req_pipe
    reqs, images, masks = _mixed_requests()
    with pytest.raises(ValueError, match="request 1: mask image is 96x512"):
        pipe.riffuse_requests(reqs[:2], images[:2], [None, _mask(96)])
    with pytest.raises(ValueError, match="max_batch"):
        pipe.riffuse_requests(reqs[:2], images[:2], masks[:2], max_batch=0)
    with pytest.raises(ValueError, match="one seed image"):
        pipe.riffuse_requests(reqs[:2], images[:1], masks[:2])
    long_guided = reqs[4].__class__(alpha=0.5, num_inference_steps=10, start=reqs[4].start.__class__(
        prompt=LONG_PROMPT, seed=1, guidance=7.0), end=reqs[4].end.__class__(prompt=LONG_PROMPT, seed=2, guidance=7.0))
    with pytest.raises(ValueError, match="request 1: the prompts embed to 154 tokens; guidance 7.0 needs 77"):
        pipe.riffuse_requests([reqs[0], long_guided], images[:2], [None, None])
    uneven = reqs[4].__class__(alpha=0.5, num_inference_steps=10, start=reqs[4].start,
                               end=reqs[0].end.__class__(prompt="short", seed=2, guidance=1.0))
    with pytest.raises(ValueError, match="request 0: the start and end prompts embed to 154 and 77 tokens"):
        pipe.riffuse_requests([uneven], images[:1], [None])
    assert pipe.context_error(reqs[4]) is None and pipe.context_error(reqs[0]) is None
    for cls in (DPMSolverMultistepSchedulerB200, EulerAncestralSchedulerB200):
        pipe.scheduler = cls()
        with pytest.raises(ValueError, match="PNDM or DDIM"):
            pipe.riffuse_requests(reqs[:2], images[:2], masks[:2])
    assert not pipe.unet.calls


def test_riffuse_requests_ddim(req_pipe):
    from riffusion.scheduler_b200 import DDIMSchedulerB200

    pipe = req_pipe
    pipe.scheduler = DDIMSchedulerB200()
    reqs, images, masks = _mixed_requests()
    outs = pipe.riffuse_requests(reqs[:5], images[:5], masks[:5], max_batch=4)
    for i in range(5):
        assert np.array_equal(outs[i]["image"].numpy(), np.asarray(pipe.riffuse(reqs[i], images[i], masks[i]))), i


# ----------------------------------------------------------------------------------------------- compute_requests
GOLDEN = Path(__file__).parent / "golden"
SINE = (3000 * np.sin(2 * np.pi * 440 * np.arange(int(44100 * 5.11)) / 44100)).astype(np.float32)


class _Pipe:
    """records riffuse / riffuse_requests; the image is the seed image; prompts starting with "long" cannot be joined"""
    device = "cpu"

    def __init__(self):
        self.calls = []

    def riffuse(self, inputs, init_image, mask_image=None):
        return init_image.copy()

    def context_error(self, inputs):
        return "154 tokens" if inputs.start.prompt.startswith("long") else None

    def riffuse_requests(self, inputs, init_images, mask_images, *, max_batch, waveform):
        self.calls.append((list(inputs), [m is not None for m in mask_images], max_batch, waveform))
        return [dict(image=torch.from_numpy(np.array(im)), waveform=None) for im in init_images]


def _seed_dir(tmp_path):
    rgb = np.load(GOLDEN / "og_beat.npz")["rgb"]
    Image.fromarray(rgb, mode="RGB").save(tmp_path / "og_beat.png")
    Image.fromarray(np.full((512, 512), 255, np.uint8), mode="L").save(tmp_path / "mask_all.png")
    Image.fromarray(np.full((512, 256), 255, np.uint8), mode="L").save(tmp_path / "mask_small.png")
    Image.fromarray(rgb[:256], mode="RGB").save(tmp_path / "short.png")
    return tmp_path


@pytest.fixture
def stub_converter(monkeypatch):
    """the real SpectrogramImageConverter over a host stand-in for inverse mel + Griffin-Lim, which draws its phases as
    the real one does; returns the list of its (mel, phases) calls"""
    from riffusion import server
    from riffusion.spectrogram_converter import SpectrogramConverter
    from riffusion.spectrogram_image_converter import SpectrogramImageConverter

    calls = []

    class _Spec(SpectrogramConverter):
        def __init__(self, params):
            self.p, self.device = params, "cpu"

        def waveform_from_mel_amplitudes(self, mel, init_angles=None):
            m = mel.reshape(-1, *mel.shape[-2:])
            F = self.p.n_fft // 2 + 1
            if init_angles is None:
                init_angles = torch.rand((m.shape[0], F, m.shape[-1]), dtype=torch.complex64, device=m.device)
            ang = init_angles.reshape(m.shape[0], F, m.shape[-1])
            calls.append((mel.clone(), init_angles.clone()))
            t = torch.arange(self.p.hop_length * (m.shape[-1] - 1), dtype=torch.float32)
            # row by row: each clip's bits do not depend on its batch, as the kernel's (tests/test_audio_gpu.py)
            w = torch.stack([3000 * torch.sin(t / 7.0) * (1 + 1e-9 * m[k].mean()) + 100 * ang[k].real.mean()
                             for k in range(m.shape[0])])
            return w.reshape(*mel.shape[:-2], -1)

    class _Conv(SpectrogramImageConverter):
        def __init__(self, params, device):
            self.p, self.device, self.converter = params, device, _Spec(params)

    monkeypatch.setattr(server, "SpectrogramImageConverter", _Conv)
    return calls


def _payload(**kw):
    p = {"alpha": 0.25, "num_inference_steps": 50, "seed_image_id": "og_beat",
         "start": {"prompt": "church bells on sunday", "seed": 42}, "end": {"prompt": "jazz with piano", "seed": 123}}
    p.update(kw)
    return p


def test_compute_requests_responses_and_refusals(tmp_path, stub_converter):
    """400s for that request only; every other response is byte for byte what sequential compute_request calls return
    under the same torch.manual_seed (same mel, same phases, same host tail); Griffin-Lim runs once per batch"""
    from riffusion import server
    from riffusion.datatypes import InferenceInput

    seed = _seed_dir(tmp_path)
    payloads = [_payload(), _payload(seed_image_id="nope"), _payload(mask_image_id="mask_all", alpha=0.5),
                _payload(mask_image_id="nope"), _payload(mask_image_id="mask_small"), _payload(alpha=1.0),
                _payload(seed_image_id="short"), _payload(start={"prompt": "long prompt", "seed": 1}),
                _payload(alpha=0.75)]
    inputs = [InferenceInput.from_dict(p) for p in payloads]
    pipe = _Pipe()
    torch.manual_seed(0)
    got = server.compute_requests(inputs, pipe, str(seed), max_batch=4)
    batched_calls = list(stub_converter)
    assert got[1] == ("Invalid seed image: nope", 400) and got[3] == ("Invalid mask image: nope", 400)
    assert got[4][1] == 400 and "mask_small is 256x512" in got[4][0]
    assert got[6][1] == 400 and "256 pixels high" in got[6][0]
    assert got[7] == ("Invalid prompts: 154 tokens", 400)
    (batch, masked, max_batch, waveform), = pipe.calls
    assert [r.alpha for r in batch] == [0.25, 0.5, 1.0, 0.75] and masked == [False, True, False, False]
    assert max_batch == 4 and waveform is False
    assert len(batched_calls) == 1 and batched_calls[0][0].shape == (4, 1, 512, 512)
    stub_converter.clear()
    torch.manual_seed(0)
    for i in (0, 2, 5, 8):
        assert got[i] == server.compute_request(inputs[i], pipe, str(seed)), i
        assert set(json.loads(got[i])) == {"image", "audio", "duration_s"}
    assert torch.equal(torch.stack([c[1] for c in stub_converter]), batched_calls[0][1])       # the same phases
    assert torch.equal(torch.stack([c[0] for c in stub_converter]), batched_calls[0][0])       # the same host mel
    assert server.compute_requests(inputs[1:2], pipe, str(seed)) == [("Invalid seed image: nope", 400)]
    assert len(pipe.calls) == 1


# ----------------------------------------------------------------------------------------------- InferenceBatcher
class _Gate:
    """stands in for compute_requests: records each batch, answers each request with its alpha, raises for alpha 0.99,
    and can be held shut so that requests pile up"""

    def __init__(self):
        self.batches = []
        self.open = threading.Event()
        self.open.set()
        self.entered = threading.Event()

    def __call__(self, inputs_list, pipeline, seed_images_dir, *, max_batch):
        self.entered.set()
        self.open.wait(10)
        self.batches.append([i.alpha for i in inputs_list])
        if any(i.alpha == 0.99 for i in inputs_list):
            raise RuntimeError("boom")
        return [f"alpha={i.alpha}" for i in inputs_list]


@pytest.fixture
def gate(monkeypatch):
    from riffusion import server

    g = _Gate()
    monkeypatch.setattr(server, "compute_requests", g)
    return g


def _workers():
    return [t for t in threading.enumerate() if t.name == "InferenceBatcher"]


def test_batcher_respects_max_batch_and_resolves_each_future(gate):
    from riffusion.server import InferenceBatcher

    with InferenceBatcher(None, "/nowhere", max_batch=4, max_wait_s=0.05) as b:
        gate.open.clear()
        first = b.submit(_payload(alpha=0.0))
        assert gate.entered.wait(5)                     # the first batch is running; the next 10 queue behind it
        futs = [b.submit(_payload(alpha=round(0.01 * (k + 1), 2))) for k in range(10)]
        gate.open.set()
        assert first.result(5) == "alpha=0.0"
        for k, f in enumerate(futs):
            assert f.result(5) == f"alpha={round(0.01 * (k + 1), 2)}"
    assert gate.batches[0] == [0.0] and [len(x) for x in gate.batches[1:]] == [4, 4, 2]
    assert b.batch_sizes == [1, 4, 4, 2]
    assert not _workers()


def test_batcher_waits_max_wait_s_for_company(gate):
    from riffusion.server import InferenceBatcher

    with InferenceBatcher(None, "/nowhere", max_batch=8, max_wait_s=0.3) as b:
        t0 = time.monotonic()
        f1 = b.submit(_payload(alpha=0.1))
        time.sleep(0.05)
        f2 = b.submit(_payload(alpha=0.2))
        assert (f1.result(5), f2.result(5)) == ("alpha=0.1", "alpha=0.2")
        assert time.monotonic() - t0 >= 0.3
        assert gate.batches == [[0.1, 0.2]]
    with InferenceBatcher(None, "/nowhere", max_batch=2, max_wait_s=30.0) as b:
        t0 = time.monotonic()
        fs = [b.submit(_payload(alpha=a)) for a in (0.1, 0.2)]
        assert [f.result(5) for f in fs] == ["alpha=0.1", "alpha=0.2"]
        assert time.monotonic() - t0 < 10                # a full batch does not wait out max_wait_s
    assert not _workers()


def test_batcher_exception_reaches_its_batch_only(gate):
    from riffusion.server import InferenceBatcher

    with InferenceBatcher(None, "/nowhere", max_batch=8, max_wait_s=0.2) as b:
        bad = [b.submit(_payload(alpha=a)) for a in (0.5, 0.99)]
        for f in bad:
            with pytest.raises(RuntimeError, match="boom"):
                f.result(5)
        assert b.submit(_payload(alpha=0.7)).result(5) == "alpha=0.7"     # the worker carries on
    assert not _workers()


def test_batcher_survives_a_cancelled_future(gate):
    """a future cancelled while it waits is dropped from its batch; the worker carries on, later requests are
    answered, and close() joins"""
    from riffusion.server import InferenceBatcher

    b = InferenceBatcher(None, "/nowhere", max_batch=8, max_wait_s=0.05)
    gate.open.clear()
    first = b.submit(_payload(alpha=0.1))
    assert gate.entered.wait(5)
    gone = b.submit(_payload(alpha=0.2))
    kept = b.submit(_payload(alpha=0.3))
    assert gone.cancel()
    gate.open.set()
    assert (first.result(5), kept.result(5)) == ("alpha=0.1", "alpha=0.3")
    assert b.submit(_payload(alpha=0.4)).result(5) == "alpha=0.4"
    alone = b.submit(_payload(alpha=0.5))
    gate.open.clear()
    time.sleep(0.01)
    alone.cancel()                                 # maybe too late: then it is answered, else never computed
    gate.open.set()
    b.close()
    assert not _workers()
    assert [0.2] not in gate.batches and all(0.2 not in x for x in gate.batches)
    assert alone.cancelled() or alone.result(0) == "alpha=0.5"


def test_batcher_parse_error_close_and_submit_after_close(gate):
    from riffusion.server import InferenceBatcher

    b = InferenceBatcher(None, "/nowhere", max_batch=8, max_wait_s=0.5)
    assert len(_workers()) == 1
    bad = b.submit({"alpha": 0.5, "start": {"prompt": "x"}})
    assert bad.done() and bad.result()[1] == 400
    queued = [b.submit(_payload(alpha=a)) for a in (0.1, 0.2, 0.3)]
    b.close()                                          # drains the queue, then joins
    assert [f.result(0) for f in queued] == ["alpha=0.1", "alpha=0.2", "alpha=0.3"]
    assert not _workers()
    with pytest.raises(RuntimeError, match="closed"):
        b.submit(_payload())
    b.close()
    with pytest.raises(ValueError, match="max_batch"):
        InferenceBatcher(None, "/nowhere", max_batch=0)


# ----------------------------------------------------------------------------------------------- operand contract
def _lat(*lead):
    return torch.zeros((*lead, 4, 8, 8), dtype=torch.float16)


def _rows(b):
    return torch.zeros((b, 13), dtype=torch.int32)


def VALID():
    return (_lat(4), _rows(2), _lat(4, 2), _lat(2), _lat(2), _lat(2), _lat(2), _lat(2), 0.5, 0.8)


def _with(k, v):
    args = list(VALID())
    args[k] = v
    return tuple(args)


MALFORMED = {
    "eps_pair_rows": lambda: _with(0, _lat(2)),
    "rows_count": lambda: _with(1, _rows(3)),
    "ring_slots": lambda: _with(2, _lat(3, 2)),
    "saved_shape": lambda: _with(3, _lat(1)),
    "sample_dtype": lambda: _with(4, _lat(2).float()),
    "init_dtype": lambda: _with(5, _lat(2).float()),
    "init_shape": lambda: _with(5, _lat(1)),
    "noise_shape": lambda: _with(6, _lat(3)),
    "noise_strided": lambda: _with(6, _lat(4)[::2]),
    "mask_dtype": lambda: _with(7, _lat(2).bool()),
    "mask_shape": lambda: _with(7, _lat(1)),
}


def test_rows_mask_step_contract(monkeypatch):
    from riffusion import _native
    from riffusion.scheduler_b200 import cfg_pndm_rows_mask_step

    calls = []
    monkeypatch.setattr(_native, "is_device_tensor", lambda t: t.device.type == "cpu")
    monkeypatch.setattr(_native, "call", lambda name, device, *args: calls.append((name, args)))
    prev = cfg_pndm_rows_mask_step(*VALID())
    assert [c[0] for c in calls] == ["rf_cfg_pndm_rows_mask_step_f16"] and calls[0][1][1:3] == (2, 256)
    assert calls[0][1][-3:-1] == (0.5, 0.8)
    assert prev.shape == (2, 4, 8, 8) and prev.dtype == torch.float16
    for name, run in MALFORMED.items():
        calls.clear()
        with pytest.raises((ValueError, _native.NativeError)):
            cfg_pndm_rows_mask_step(*run())
        assert calls == [], name


def test_rows_mask_step_refuses_host_tensors(monkeypatch):
    from riffusion import _native
    from riffusion.scheduler_b200 import cfg_pndm_rows_mask_step

    calls = []
    monkeypatch.setattr(_native, "call", lambda name, device, *args: calls.append(name))
    with pytest.raises(_native.NativeError, match="CUDA tensor"):
        cfg_pndm_rows_mask_step(*VALID())
    assert calls == []


# ----------------------------------------------------------------------------------------------- bench
def test_bench_server_accounting():
    spec = importlib.util.spec_from_file_location("bench_server", ROOT / "tools" / "bench_server.py")
    mod = importlib.util.module_from_spec(spec)
    sys.modules["bench_server"] = mod
    spec.loader.exec_module(mod)
    from riffusion.datatypes import InferenceInput, PromptInput

    def req(alpha, den=0.75, g=7.0):
        return InferenceInput(alpha=alpha, num_inference_steps=50, start=PromptInput(prompt="a", seed=1, denoising=den,
                                                                                     guidance=g),
                              end=PromptInput(prompt="b", seed=2, denoising=den, guidance=g))

    one = mod.loop_accounting([req(0.0)], 16)
    assert one == {"loops": 1, "requests": 1, "unet_evals": 38, "cfg_batch": [2], "rows": 1, "filler_rows": 0,
                   "row_evals": 38, "filler_fraction": 0.0}
    five = mod.loop_accounting([req(a) for a in (0.0, 0.25, 0.5, 0.75, 1.0)], 16)
    assert five["loops"] == 1 and five["cfg_batch"] == [16] and five["filler_rows"] == 3
    assert five["unet_evals"] == 38 and five["row_evals"] == 8 * 38 and five["filler_fraction"] == 3 / 8
    mixed = mod.loop_accounting([req(0.5, 0.5), req(0.5, 0.9), req(0.0, 0.75, 1.0)], 16)
    assert mixed["loops"] == 2 and mixed["cfg_batch"] == [4, 1] and mixed["unet_evals"] == 46 + 38
    assert mod.loop_accounting([req(0.0)] * 20, 16)["cfg_batch"] == [32, 8]
    # the serial arm: one loop per request at CFG batch 2
    assert mod.serial_accounting([req(0.0), req(0.5, 0.5)]) == {"loops": 2, "unet_evals": 38 + 26, "cfg_batch": [2, 2]}
