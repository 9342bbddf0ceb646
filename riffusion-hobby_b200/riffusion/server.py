"""Inference request -> JSON response, the model server's contract without the web framework
(reference: riffusion/server.py:66-183; Flask itself is outside SURVEY §8 and not installed here).

`compute_request(inputs, pipeline, seed_images_dir)` keeps the reference's signature and return convention: a JSON string
of `InferenceOutput` on success, or a `(message, 400)` tuple for a bad seed / mask id.  `run_inference(json_data, ...)`
is the body of the `/run_inference/` route (:83-112) operating on an already-parsed JSON object.

Concurrent clients: `compute_requests(inputs_list, ...)` answers many requests with `RiffusionPipeline.riffuse_requests`
(one CFG loop per group of compatible requests instead of one loop per request) and returns what `compute_request`
would return for each.  `InferenceBatcher` gathers requests submitted from many threads into such batches on one worker
thread that owns the pipeline; a web route would call `batcher.submit(request.json).result()`.

What differs, loudly:
  * audio container: the reference exports MP3 through pydub + ffmpeg (:166-169).  Neither exists in this image; when the
    segment cannot export "mp3" the response carries `data:audio/wav;base64,...` instead (same int16 PCM, lossless).
  * between `riffuse` and the audio the reference goes GPU -> PIL -> numpy -> GPU; `fast_audio=True` (default when the
    pipeline offers `generate_clips`-style device glue) keeps that on the device but returns byte-identical JSON fields.
"""
from __future__ import annotations

import concurrent.futures
import dataclasses
import io
import json
import logging
import queue
import threading
import time
import typing as T
from pathlib import Path

import numpy as np
import PIL.Image
import torch

from riffusion.datatypes import InferenceInput, InferenceOutput
from riffusion.spectrogram_image_converter import SpectrogramImageConverter
from riffusion.spectrogram_params import SpectrogramParams
from riffusion.util import base64_util

SEED_IMAGES_DIR = Path(Path(__file__).resolve().parent.parent, "seed_images")


def run_inference(json_data: T.Mapping[str, T.Any], pipeline, seed_images_dir: T.Union[str, Path] = SEED_IMAGES_DIR):
    """parse + validate the request like the route does (dacite errors -> 400), then `compute_request`"""
    start_time = time.time()
    try:
        inputs = InferenceInput.from_dict(json_data)
    except (TypeError, KeyError, ValueError) as exception:          # dacite WrongTypeError / MissingValueError
        logging.info(json_data)
        return str(exception), 400
    response = compute_request(inputs=inputs, seed_images_dir=str(seed_images_dir), pipeline=pipeline)
    logging.info(f"Request took {time.time() - start_time:.2f} s")
    return response


def compute_request(inputs: InferenceInput, pipeline, seed_images_dir: str) -> T.Union[str, T.Tuple[str, int]]:
    init_image_path = Path(seed_images_dir, f"{inputs.seed_image_id}.png")
    if not init_image_path.is_file():
        return f"Invalid seed image: {inputs.seed_image_id}", 400
    init_image = PIL.Image.open(str(init_image_path)).convert("RGB")

    mask_image: T.Optional[PIL.Image.Image] = None
    if inputs.mask_image_id:
        mask_image_path = Path(seed_images_dir, f"{inputs.mask_image_id}.png")
        if not mask_image_path.is_file():
            return f"Invalid mask image: {inputs.mask_image_id}", 400
        mask_image = PIL.Image.open(str(mask_image_path)).convert("RGB")

    image = pipeline.riffuse(inputs, init_image=init_image, mask_image=mask_image)

    params = SpectrogramParams(min_frequency=0, max_frequency=10000)
    converter = SpectrogramImageConverter(params=params, device=str(pipeline.device))    # plans are cached per geometry
    segment = converter.audio_from_spectrogram_image(image, apply_filters=True)
    return _response(image, segment)


def _response(image: PIL.Image.Image, segment) -> str:
    """The JSON of `InferenceOutput`: the segment as MP3 (WAV where MP3 cannot be written) and the image as JPEG, both
    base64 data URLs."""
    audio_bytes = io.BytesIO()
    try:
        segment.export(audio_bytes, format="mp3")
        audio_mime = "audio/mpeg"
    except (NotImplementedError, ValueError, OSError):
        audio_bytes = io.BytesIO()
        segment.export(audio_bytes, format="wav")
        audio_mime = "audio/wav"
    audio_bytes.seek(0)

    image_bytes = io.BytesIO()
    image.save(image_bytes, exif=image.getexif(), format="JPEG")
    image_bytes.seek(0)

    output = InferenceOutput(
        image="data:image/jpeg;base64," + base64_util.encode(image_bytes),
        audio=f"data:{audio_mime};base64," + base64_util.encode(audio_bytes),
        duration_s=segment.duration_seconds,
    )
    return json.dumps(dataclasses.asdict(output))


def _load_request(inputs: InferenceInput, seed_images_dir: str, num_frequencies: int):
    """(seed image, mask image or None) of a request as `compute_request` opens them, or the (message, 400) it returns
    for an unknown id.  Also 400: a mask whose size differs from its seed image, and a seed image whose height (rounded
    down to a multiple of 32) is not `num_frequencies`; in a batch either would fail every request with it."""
    init_image_path = Path(seed_images_dir, f"{inputs.seed_image_id}.png")
    if not init_image_path.is_file():
        return f"Invalid seed image: {inputs.seed_image_id}", 400
    init_image = PIL.Image.open(str(init_image_path)).convert("RGB")
    mask_image: T.Optional[PIL.Image.Image] = None
    if inputs.mask_image_id:
        mask_image_path = Path(seed_images_dir, f"{inputs.mask_image_id}.png")
        if not mask_image_path.is_file():
            return f"Invalid mask image: {inputs.mask_image_id}", 400
        mask_image = PIL.Image.open(str(mask_image_path)).convert("RGB")
        if mask_image.size != init_image.size:
            return (f"Mask image {inputs.mask_image_id} is {mask_image.size[0]}x{mask_image.size[1]}, seed image "
                    f"{inputs.seed_image_id} is {init_image.size[0]}x{init_image.size[1]}"), 400
    if init_image.height - init_image.height % 32 != num_frequencies:
        return (f"Seed image {inputs.seed_image_id} is {init_image.height} pixels high; the spectrogram needs "
                f"{num_frequencies}"), 400
    return init_image, mask_image


def compute_requests(inputs_list: T.Sequence[InferenceInput], pipeline, seed_images_dir: str, *,
                     max_batch: int = 16) -> T.List[T.Union[str, T.Tuple[str, int]]]:
    """`compute_request` for many requests at once: one response per request, in order, each the JSON string or the
    (message, 400) `compute_request` would return.  Also a 400, for that request only, where `riffuse` would raise:
    a prompt pair the pipeline cannot join into one context (`pipeline.context_error`), besides `_load_request`'s.

    The valid requests run through `pipeline.riffuse_requests` (batched CFG loops, at most `max_batch` rows each).  The
    audio tail is `audio_from_spectrogram_image`'s: the host mel of each uint8 image, then inverse mel + Griffin-Lim on
    the device, batched over the requests of one width (each clip's bits do not depend on its batch), then per request
    peak-normalised int16, `apply_filters`, MP3 (or WAV) and the JPEG.  Griffin-Lim's initial phases are drawn per valid
    request, in request order, with the shape, RNG and dtype `audio_from_spectrogram_image` uses, so under one
    torch.manual_seed each response is byte for byte the one sequential `compute_request` calls would return, given
    the same image."""
    from riffusion.util import audio_util, image_util

    params = SpectrogramParams(min_frequency=0, max_frequency=10000)
    responses: T.List[T.Any] = [None] * len(inputs_list)
    valid, images, masks = [], [], []
    for i, inputs in enumerate(inputs_list):
        loaded = _load_request(inputs, seed_images_dir, params.num_frequencies)
        if isinstance(loaded[1], int):
            responses[i] = loaded
            continue
        error = pipeline.context_error(inputs)
        if error is not None:
            responses[i] = f"Invalid prompts: {error}", 400
            continue
        valid.append(i)
        images.append(loaded[0])
        masks.append(loaded[1])
    if not valid:
        return responses
    channels = 2 if params.stereo else 1
    angles = [torch.rand((channels, params.n_fft // 2 + 1, img.width - img.width % 32), dtype=torch.complex64,
                         device=pipeline.device) for img in images]
    outs = pipeline.riffuse_requests([inputs_list[i] for i in valid], images, masks, max_batch=max_batch,
                                     waveform=False)
    pils = [PIL.Image.fromarray(out["image"].cpu().numpy()) for out in outs]
    mels = [image_util.spectrogram_from_image(im, max_value=30e6, power=params.power_for_image, stereo=params.stereo)
            for im in pils]
    converter = SpectrogramImageConverter(params=params, device=str(pipeline.device)).converter
    waves: T.List[T.Any] = [None] * len(valid)
    for width in sorted({m.shape[-1] for m in mels}):
        ks = [k for k, m in enumerate(mels) if m.shape[-1] == width]
        mel = torch.from_numpy(np.stack([mels[k] for k in ks])).to(pipeline.device)
        wave = converter.waveform_from_mel_amplitudes(mel, torch.stack([angles[k] for k in ks])).cpu().numpy()
        for j, k in enumerate(ks):
            waves[k] = wave[j]
    for k, i in enumerate(valid):
        segment = audio_util.audio_from_waveform(samples=waves[k], sample_rate=params.sample_rate, normalize=True)
        responses[i] = _response(pils[k], audio_util.apply_filters(segment, compression=False))
    return responses


class InferenceBatcher:
    """Coalesces `/run_inference/` requests from many threads into `compute_requests` batches.

    `submit(json_data)` parses the request like `run_inference` and returns a Future of its response (a parse error
    resolves it at once to (message, 400)).  One worker thread owns the pipeline and all GPU work: it takes the first
    waiting request, collects more for up to `max_wait_s` or until `max_batch` are waiting, and answers them with one
    `compute_requests` call; requests that arrive meanwhile wait for the next batch.  A future cancelled before its
    batch starts is dropped from it.  An exception inside a batch is set on every future of that batch and the worker
    carries on.  `close()` answers what is queued, then joins the worker;
    `submit` after `close` raises RuntimeError.  Usable as a context manager."""

    def __init__(self, pipeline, seed_images_dir: T.Union[str, Path] = SEED_IMAGES_DIR, *, max_batch: int = 16,
                 max_wait_s: float = 0.02):
        if max_batch < 1:
            raise ValueError("max_batch must be at least 1")
        self.pipeline, self.seed_images_dir = pipeline, str(seed_images_dir)
        self.max_batch, self.max_wait_s = max_batch, max_wait_s
        self.batch_sizes: T.List[int] = []
        self._queue: "queue.Queue[T.Optional[T.Tuple[InferenceInput, concurrent.futures.Future]]]" = queue.Queue()
        self._lock = threading.Lock()
        self._closed = False
        self._worker = threading.Thread(target=self._run, name="InferenceBatcher", daemon=True)
        self._worker.start()

    def submit(self, json_data: T.Mapping[str, T.Any]) -> concurrent.futures.Future:
        future: concurrent.futures.Future = concurrent.futures.Future()
        with self._lock:
            if self._closed:
                raise RuntimeError("InferenceBatcher is closed")
            try:
                inputs = InferenceInput.from_dict(json_data)
            except (TypeError, KeyError, ValueError) as exception:          # as run_inference
                logging.info(json_data)
                future.set_result((str(exception), 400))
                return future
            self._queue.put((inputs, future))
        return future

    def _run(self) -> None:
        while True:
            first = self._queue.get()
            if first is None:
                return
            batch = [first]
            stop = False
            deadline = time.monotonic() + self.max_wait_s
            while len(batch) < self.max_batch:
                try:
                    item = self._queue.get(timeout=max(0.0, deadline - time.monotonic()))
                except queue.Empty:
                    break
                if item is None:
                    stop = True
                    break
                batch.append(item)
            # a future its caller cancelled (a timeout, a disconnected client) is dropped; the others can no longer be
            # cancelled, so setting their result below cannot fail
            batch = [(inputs, future) for inputs, future in batch if future.set_running_or_notify_cancel()]
            if batch:
                self._answer(batch)
            if stop:
                return

    def _answer(self, batch) -> None:
        self.batch_sizes.append(len(batch))
        try:
            responses = compute_requests([inputs for inputs, _ in batch], self.pipeline, self.seed_images_dir,
                                         max_batch=self.max_batch)
        except Exception as exception:                                    # noqa: BLE001 - handed to every caller
            for _, future in batch:
                future.set_exception(exception)
        else:
            for (_, future), response in zip(batch, responses):
                future.set_result(response)

    def close(self) -> None:
        """Answer every queued request, then stop and join the worker.  Idempotent."""
        with self._lock:
            if self._closed:
                return
            self._closed = True
            self._queue.put(None)
        self._worker.join()

    def __enter__(self) -> "InferenceBatcher":
        return self

    def __exit__(self, *exc) -> None:
        self.close()
