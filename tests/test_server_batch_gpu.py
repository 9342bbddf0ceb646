"""The batched model server on the H100: `rf_cfg_pndm_rows_mask_step_f16` against fp64 and against the rows step
followed by `rf_axpby_f16`, one-request batches against `compute_request`, a heterogeneous batch against per-request
`riffuse`, graph replay, `max_batch`, and concurrent clients through `InferenceBatcher`."""
import base64
import io
import json
import threading

import numpy as np
import pytest
import torch
from PIL import Image

from test_interpolation_gpu import _close, _seed_image, _table
from test_text_to_audio_gpu import _t2a_pipe, vae_pair  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu


def _records():
    """every kind of record, masked and not, pushing to and reading from every ring slot"""
    from riffusion.scheduler_b200 import ROW_BASE_SAVED, ROW_MASK, ROW_SAVE

    return [
        dict(active=0, guidance=7.0, flags=ROW_MASK),
        dict(active=1, guidance=3.5, c0=1.0, ca=0.97, cb=0.11, push=0, flags=ROW_SAVE | ROW_MASK),
        dict(active=1, guidance=0.0, c0=0.5, c1=0.5, h1=2, ca=1.02, cb=0.2, flags=ROW_BASE_SAVED),
        dict(active=1, guidance=9.25, c0=1.5, c1=-0.5, h1=3, ca=0.99, cb=0.05, push=1, flags=ROW_MASK),
        dict(active=1, guidance=1.75, c0=23 / 12, c1=-16 / 12, c2=5 / 12, h1=0, h2=1, ca=1.01, cb=0.3, push=2),
        dict(active=1, guidance=5.0, c0=55 / 24, c1=-59 / 24, c2=37 / 24, c3=-9 / 24, h1=3, h2=2, h3=0, ca=0.95,
             cb=0.07, push=3, flags=ROW_MASK),
        dict(active=0, guidance=12.0, push=3, flags=ROW_SAVE),
        dict(active=1, guidance=7.0, c0=0.5, c1=0.5, h1=1, ca=1.0, cb=0.1, flags=ROW_BASE_SAVED | ROW_MASK),
    ]


def _inputs(shape, seed):
    torch.manual_seed(seed)
    B = shape[0]
    pair = torch.randn((2 * B,) + shape[1:], device="cuda").half()
    x = (torch.randn(shape, device="cuda") * 2).half()
    ring = torch.randn((4,) + shape, device="cuda").half()
    saved = torch.randn(shape, device="cuda").half()
    init = torch.randn(shape, device="cuda").half()
    noise = torch.randn(shape, device="cuda").half()
    mask = torch.rand(shape, device="cuda").half()
    mask[:, :, :2] = (mask[:, :, :2] > 0.5).half()                  # hard 0 / 1 and soft values
    return pair, x, ring, saved, init, noise, mask


def _nan_unblended(recs, init, noise, mask):
    from riffusion.scheduler_b200 import ROW_MASK

    for r, rec in enumerate(recs):
        if not (rec["active"] and rec.get("flags", 0) & ROW_MASK):
            init[r], noise[r], mask[r] = float("nan"), float("nan"), float("nan")


@torch.no_grad()
def test_mask_kernel_against_fp64(native_lib):
    """mixed records: active, inactive, masked, unmasked, every ring slot; an odd element count per row.  Within one
    fp16 rounding plus 2^-20 relative of fp64; the NaN blend inputs of the other rows never reach the output"""
    from riffusion.scheduler_b200 import ROW_BASE_SAVED, ROW_MASK, cfg_pndm_rows_mask_step

    recs = _records()
    shape = (len(recs), 4, 9, 13)
    pair, x, ring, saved, init, noise, mask = _inputs(shape, 21)
    _nan_unblended(recs, init, noise, mask)
    B = shape[0]
    a, b = 0.8125, 0.5830951894845301
    ring0, saved0 = ring.clone(), saved.clone()
    prev = cfg_pndm_rows_mask_step(pair, _table(B, recs), ring, saved, x, init, noise, mask, a, b)
    assert not torch.isnan(prev).any()
    f = lambda v: float(np.float32(v))          # noqa: E731  (the C floats the kernel reads)
    eu, et = pair[:B], pair[B:]
    for r, rec in enumerate(recs):
        if not rec["active"]:
            assert torch.equal(prev[r], x[r])
            continue
        e0 = (eu[r] + ((et[r] - eu[r]).float() * f(rec["guidance"])).half()).double()
        e = f(rec["c0"]) * e0
        for c, h in (("c1", "h1"), ("c2", "h2"), ("c3", "h3")):
            if rec.get(h, -1) >= 0:
                e = e + f(rec[c]) * ring0[rec[h], r].double()
        base = saved0[r] if rec.get("flags", 0) & ROW_BASE_SAVED else x[r]
        want = f(rec["ca"]) * base.double() - f(rec["cb"]) * e
        if rec.get("flags", 0) & ROW_MASK:
            p = want.half().double()                                   # the stepped value is rounded first
            m = mask[r].double()
            want = (f(a) * init[r].double() + f(b) * noise[r].double()) * m + p * (1 - m)
        err = (prev[r].double() - want).abs()
        tol = want.abs() * (2 ** -11 + 2 ** -20) + 2 ** -24 + 2 ** -20 * (want.abs().max() + 1)
        if rec.get("flags", 0) & ROW_MASK:
            tol = tol + p.abs() * 2 ** -10                                # ... and p's own rounding
        assert (err <= tol).all(), (r, float(err.max()))


@torch.no_grad()
def test_mask_kernel_bits(native_lib):
    """a table without mask flags gives rf_cfg_pndm_rows_step_f16's bits; every masked row gives the bits of
    rf_cfg_pndm_rows_step_f16 followed by rf_axpby_f16; NaN in the other rows' blend inputs changes nothing"""
    from riffusion import tc_ops
    from riffusion.scheduler_b200 import ROW_MASK, cfg_pndm_rows_mask_step, cfg_pndm_rows_step

    recs = _records()
    shape = (len(recs), 4, 32, 24)
    B = shape[0]
    a, b = 0.9531, 0.3027
    for trial in range(3):
        pair, x, ring, saved, init, noise, mask = _inputs(shape, 40 + trial)
        plain_recs = [dict(rec, flags=rec.get("flags", 0) & ~ROW_MASK) for rec in recs]
        ring_p, saved_p = ring.clone(), saved.clone()
        want = cfg_pndm_rows_step(pair, _table(B, plain_recs), ring_p, saved_p, x)
        nan_init, nan_noise, nan_mask = init.clone(), noise.clone(), mask.clone()
        _nan_unblended(recs, nan_init, nan_noise, nan_mask)
        ring_m, saved_m = ring.clone(), saved.clone()
        got_plain = cfg_pndm_rows_mask_step(pair, _table(B, plain_recs), ring.clone(), saved.clone(), x, nan_init,
                                            nan_noise, nan_mask, a, b)
        assert torch.equal(got_plain, want)
        got = cfg_pndm_rows_mask_step(pair, _table(B, recs), ring_m, saved_m, x, nan_init, nan_noise, nan_mask, a, b)
        assert torch.equal(ring_m, ring_p) and torch.equal(saved_m, saved_p)
        blended = tc_ops.axpby(init, noise, a, b, mask, want)
        for r, rec in enumerate(recs):
            expect = blended[r] if rec["active"] and rec.get("flags", 0) & ROW_MASK else want[r]
            assert torch.equal(got[r], expect), (trial, r)


# ----------------------------------------------------------------------------------------------- the server
def _seed_dir(tmp_path, width=256):
    _seed_image(width, seed=4).save(tmp_path / "seed.png")
    _seed_image(width, seed=5).save(tmp_path / "seed2.png")
    m = np.zeros((512, width), np.uint8)
    m[:, width // 2:] = 255
    Image.fromarray(m, mode="L").save(tmp_path / "mask.png")
    return str(tmp_path)


def _payload(alpha=0.25, mask=None, seed_image="seed", d0=0.75, d1=0.75, g0=7.0, g1=7.0, s0=42, s1=123, steps=10):
    p = {"alpha": alpha, "num_inference_steps": steps, "seed_image_id": seed_image,
         "start": {"prompt": "church bells on sunday", "seed": s0, "denoising": d0, "guidance": g0},
         "end": {"prompt": "jazz with (piano:1.2)", "seed": s1, "denoising": d1, "guidance": g1}}
    if mask:
        p["mask_image_id"] = mask
    return p


def _pcm(resp):
    from scipy.io import wavfile

    head, data = json.loads(resp)["audio"].split(",", 1)
    assert head == "data:audio/wav;base64"
    return wavfile.read(io.BytesIO(base64.decodebytes(data.encode())))[1].astype(np.int32)


@torch.no_grad()
@pytest.mark.parametrize("mask", [None, "mask"])
def test_batch_of_one_is_compute_request(vae_pair, tmp_path, mask):
    """one request through compute_requests against compute_request under the same torch.manual_seed: the response
    JSON byte for byte"""
    from riffusion import server
    from riffusion.datatypes import InferenceInput

    _, vae = vae_pair
    pipe = _t2a_pipe(vae)
    seed = _seed_dir(tmp_path)
    inputs = InferenceInput.from_dict(_payload(alpha=0.4, mask=mask, d0=0.6, d1=0.85, g0=6.0, g1=8.0))
    torch.manual_seed(7)
    want = server.compute_request(inputs, pipe, seed)
    torch.manual_seed(7)
    got, = server.compute_requests([inputs], pipe, seed)
    assert got == want


@torch.no_grad()
def test_batch_audio_is_compute_requests_audio_path(vae_pair, tmp_path):
    """a batch over two seed-image widths: each response's audio is compute_request's audio path (host mel, inverse
    mel + Griffin-Lim alone, int16, filters) applied to that request's batched image with the phases drawn in request
    order, sample for sample; a request whose prompts cannot be joined is a 400 and the others are answered"""
    from riffusion import server
    from riffusion.datatypes import InferenceInput
    from riffusion.riffusion_pipeline import DEFAULT_PARAMS
    from riffusion.util import audio_util, image_util

    _, vae = vae_pair
    pipe = _t2a_pipe(vae)
    seed = _seed_dir(tmp_path)
    _seed_image(384, seed=6).save(tmp_path / "wide.png")
    long_prompt = " ".join(f"word{i}" for i in range(90))
    payloads = [_payload(0.0, "mask", "seed"), _payload(0.5, None, "wide", s0=5), _payload(1.0, None, "seed2", s1=9),
                dict(_payload(0.5), start={"prompt": long_prompt, "seed": 1, "guidance": 7.0}),
                _payload(0.25, None, "wide", d0=0.9)]
    inputs = [InferenceInput.from_dict(p) for p in payloads]
    images = []
    real = pipe.riffuse_requests

    def spy(*a, **kw):
        outs = real(*a, **kw)
        images.extend(o["image"].cpu().numpy() for o in outs)
        return outs

    pipe.riffuse_requests = spy
    torch.manual_seed(11)
    got = server.compute_requests(inputs, pipe, seed)
    assert got[3][1] == 400 and got[3][0].startswith("Invalid prompts: ") and len(images) == 4
    torch.manual_seed(11)
    F = DEFAULT_PARAMS.n_fft // 2 + 1
    angles = [torch.rand((1, F, im.shape[1]), dtype=torch.complex64, device="cuda") for im in images]
    conv = pipe._converter(DEFAULT_PARAMS, None)
    for k, i in enumerate((0, 1, 2, 4)):
        mel = image_util.spectrogram_from_image(Image.fromarray(images[k]), max_value=30e6, power=0.25, stereo=False)
        wave = conv.waveform_from_mel_amplitudes(torch.from_numpy(mel).cuda(), angles[k])
        seg = audio_util.apply_filters(audio_util.audio_from_waveform(samples=wave.cpu().numpy(), sample_rate=44100,
                                                                      normalize=True))
        want = np.asarray(seg.get_array_of_samples()).astype(np.int32)
        assert np.array_equal(_pcm(got[i]).reshape(-1), want), i


@torch.no_grad()
def test_heterogeneous_batch_graph_and_max_batch(vae_pair, tmp_path):
    """mixed alphas, denoising, guidance, two seed images, masked and unmasked rows: each image against its own riffuse
    at the batch bar, each waveform against compute_request's audio path (host mel, then the device inverse) applied to
    the batched image with the same phases; graph replay equals eager bit for bit; max_batch=1 against the default"""
    from riffusion.datatypes import InferenceInput
    from riffusion.riffusion_pipeline import DEFAULT_PARAMS
    from riffusion.util import image_util

    _, vae = vae_pair
    pipe = _t2a_pipe(vae)
    seed = _seed_dir(tmp_path)
    payloads = [_payload(0.0, "mask", "seed", 0.5, 0.9, 5.0, 9.0, 1, 2), _payload(0.25, None, "seed2", 0.75, 0.75),
                _payload(0.5, "mask", "seed", 0.6, 0.8, 6.0, 8.0, 3, 4), _payload(1.0, None, "seed", 0.5, 0.9, 9.0, 5.0),
                _payload(0.75, None, "seed2", 0.9, 0.5, 5.0, 7.0, 5, 6), _payload(0.3, "mask", "seed2", 0.7, 0.7)]
    inputs = [InferenceInput.from_dict(p) for p in payloads]
    images = [Image.open(f"{seed}/{p['seed_image_id']}.png").convert("RGB") for p in payloads]
    masks = [Image.open(f"{seed}/mask.png").convert("RGB") if p.get("mask_image_id") else None for p in payloads]
    F = DEFAULT_PARAMS.n_fft // 2 + 1
    angles = [torch.rand((1, F, 256), dtype=torch.complex64, device="cuda") for _ in inputs]
    outs = pipe.riffuse_requests(inputs, images, masks, init_angles=angles)
    assert {o["filler_rows"] for o in outs} == {2} and len({o["loop"] for o in outs}) == 1
    conv = pipe._converter(DEFAULT_PARAMS, None)
    for i, (inp, img, m) in enumerate(zip(inputs, images, masks)):
        _close(outs[i]["image"].cpu().numpy(), pipe.riffuse(inp, img, mask_image=m), f"request {i} vs riffuse")
        mel = image_util.spectrogram_from_image(Image.fromarray(outs[i]["image"].cpu().numpy()), power=0.25,
                                                stereo=False, max_value=30e6)
        ref = conv.waveform_from_mel_amplitudes(torch.from_numpy(mel).cuda(), angles[i])
        rel = float((outs[i]["waveform"] - ref).norm() / ref.norm())
        # the device mel (powf) is within ~2 ulp of the host one (numpy power); 32 Griffin-Lim iterations amplify that
        # to a few 1e-4 (4.6e-4 measured on an H100)
        assert rel < 2e-3, (i, rel)
    pipe.use_cuda_graph = False
    eager = pipe.riffuse_requests(inputs, images, masks, init_angles=angles)
    pipe.use_cuda_graph = True
    for o, e in zip(outs, eager):
        assert torch.equal(o["image"], e["image"]) and torch.equal(o["waveform"], e["waveform"])
    one = pipe.riffuse_requests(inputs, images, masks, max_batch=1)
    assert len({o["loop"] for o in one}) == len(inputs) and {o["filler_rows"] for o in one} == {0}
    _close(torch.stack([o["image"] for o in one]).cpu().numpy(), torch.stack([o["image"] for o in outs]).cpu().numpy(),
           "max_batch=1 vs default")


@torch.no_grad()
def test_concurrent_clients_through_the_batcher(vae_pair, tmp_path):
    """8 threads submit 24 requests to one InferenceBatcher: every response is a JSON answer whose image matches its
    own riffuse at the batch bar, the requests coalesce into batches, and no thread is left after close()"""
    from riffusion import server
    from riffusion.datatypes import InferenceInput

    _, vae = vae_pair
    pipe = _t2a_pipe(vae)
    seed = _seed_dir(tmp_path)
    seen = {}
    real = pipe.riffuse_requests

    def spy(inputs, *a, **kw):
        outs = real(inputs, *a, **kw)
        for inp, o in zip(inputs, outs):
            seen[(inp.alpha, inp.start.seed)] = o["image"].cpu().numpy()
        return outs

    pipe.riffuse_requests = spy
    payloads = [_payload(alpha=0.25 * (k % 5), mask="mask" if k % 3 == 0 else None, seed_image="seed2" if k % 2 else "seed",
                         d0=0.6 + 0.01 * k, s0=100 + k, s1=200 + k, g0=5.0 + 0.1 * k) for k in range(24)]
    results = [None] * 24
    with server.InferenceBatcher(pipe, seed, max_batch=8, max_wait_s=0.05) as batcher:
        def client(c):
            for k in range(c, 24, 8):
                results[k] = batcher.submit(payloads[k]).result()

        threads = [threading.Thread(target=client, args=(c,)) for c in range(8)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        sizes = list(batcher.batch_sizes)
    assert not [t for t in threading.enumerate() if t.name == "InferenceBatcher"]
    assert sum(sizes) == 24 and max(sizes) <= 8 and len(sizes) < 24, sizes
    for k, p in enumerate(payloads):
        assert isinstance(results[k], str) and set(json.loads(results[k])) == {"image", "audio", "duration_s"}
        inp = InferenceInput.from_dict(p)
        img = Image.open(f"{seed}/{p['seed_image_id']}.png").convert("RGB")
        m = Image.open(f"{seed}/mask.png").convert("RGB") if p.get("mask_image_id") else None
        _close(seen[(inp.alpha, inp.start.seed)], pipe.riffuse(inp, img, mask_image=m), f"request {k} vs riffuse")
