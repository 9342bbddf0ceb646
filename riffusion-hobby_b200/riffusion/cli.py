"""Command line front end: the six commands of the reference's `python -m riffusion.cli` (riffusion/cli.py:21-278) with
the same names, flags and defaults (`COMMANDS`, what `build_parser()` builds by default), plus this package's
`text-to-audio`, the app's text-to-audio task as a command (`EXTRA_COMMANDS`; `main` offers both sets):

    python -m riffusion.cli audio-to-image --audio clip.wav --image clip.png [--stereo] [--device cuda]
    python -m riffusion.cli image-to-audio --image clip.png --audio clip.wav
    python -m riffusion.cli print-exif --image clip.png
    python -m riffusion.cli sample-clips --audio song.wav --output-dir clips --num-clips 4
    python -m riffusion.cli audio-to-images-batch --audio-dir clips --output-dir images
    python -m riffusion.cli sample-clips-batch --audio-dir songs --output-dir clips
    python -m riffusion.cli text-to-audio --prompt "jazz with piano" --audio out.wav [--image out.png]
        [--negative-prompt ...] [--seed 42] [--num-clips 1] [--num-inference-steps 30] [--guidance 7.0] [--width 512]
        [--scheduler DPMSolverMultistepScheduler] [--use-20k] [--loop] [--checkpoint DIR] [--device cuda]
    python -m riffusion.cli audio-to-audio --audio song.wav --output riffed.wav --prompt "jazz with piano"
        [--image-dir clips] [--negative-prompt ...] [--seed 42] [--denoising 0.55] [--num-inference-steps 25]
        [--guidance 7.0] [--scheduler DPMSolverMultistepScheduler] [--start-time-s 0] [--duration-s 20]
        [--clip-duration-s 5] [--overlap-duration-s 0.2] [--prompt-b ... [--seed-b N] [--denoising-b X]]
        [--max-batch 32] [--use-20k] [--magic-mix [--kmin 0.3] [--kmax 0.5] [--mix-factor 0.5]] [--checkpoint DIR]
        [--device cuda]
    python -m riffusion.cli interpolation --prompt-a "jazz" --prompt-b "rock" --seed-image og_beat.png --output walk.wav
        [--image-dir steps] [--seed-a 42] [--seed-b 42] [--denoising-a 0.75] [--denoising-b 0.75] [--guidance 7.0]
        [--num-interpolation-steps 12] [--num-inference-steps 50] [--alpha-power 1.0] [--max-batch 32]
        [--checkpoint DIR] [--device cuda]
    python -m riffusion.cli text-to-track --prompt "lo-fi piano" --audio out.wav [--image out.png]
        [--prompt-changes "20:jazz with drums;40:hard rock"] [--negative-prompt ...] [--duration-s 30] [--seed 42]
        [--num-tracks 1] [--num-inference-steps 30] [--guidance 7.0] [--scheduler DPMSolverMultistepScheduler]
        [--window-width 512] [--stride 256] [--max-batch 32] [--use-20k] [--checkpoint DIR] [--device cuda]
    python -m riffusion.cli text-to-audio-batch --json inputs.json --output-dir out [--num-seeds 1] [--max-batch 32]
        [--audio-extension wav] [--checkpoint DIR] [--device cuda]

`--scheduler` takes DPMSolverMultistepScheduler, PNDMScheduler, DDIMScheduler or EulerAncestralDiscreteScheduler
(audio-to-audio's --magic-mix refuses the last).  `text-to-audio` loads a local diffusers-layout checkpoint directory; with `--num-clips N` > 1 clip i (seed + i) is
written to out_<seed + i>.wav / .png.  `--loop` renders seamless loops: a clip of exactly hop * width samples whose
spectrogram tiles horizontally and whose audio plays on repeat without a click.  The image carries the spectrogram parameters in its EXIF block, so
`image-to-audio` turns it back into the same audio.

Each command is a keyword-only function (callable from Python exactly like the reference's); `argh`, which the reference
uses to turn those functions into sub-commands, is not installed on the GPU image, so `build_parser` derives an
argparse sub-command per function from its signature instead.  Audio I/O goes through riffusion.util.audio_util
(pydub when present, else the WAV-only stand-in).
"""
from __future__ import annotations

import argparse
import inspect
import random
import sys
import typing as T
from multiprocessing.pool import ThreadPool
from pathlib import Path

import numpy as np
from PIL import Image

from riffusion.spectrogram_image_converter import SpectrogramImageConverter
from riffusion.spectrogram_params import SpectrogramParams
from riffusion.util import image_util
from riffusion.util.audio_util import AudioSegment

_PIL_FORMAT = {"jpg": "JPEG", "jpeg": "JPEG", "png": "PNG"}


# ------------------------------------------------------------------------------------------------ shared pieces
def _store_image(picture: Image.Image, path, fmt: str) -> None:
    """Save with the EXIF block (conversion parameters + MAX_VALUE) that image-to-audio reads back."""
    picture.save(path, exif=picture.getexif(), format=fmt)


def _store_spectrogram(pixels: np.ndarray, params: SpectrogramParams, path, fmt: str = "PNG") -> None:
    """Save a (H, W, 3) uint8 spectrogram image with `params` in its EXIF block."""
    picture = Image.fromarray(pixels)
    picture.getexif().update(params.to_exif().items())
    _store_image(picture, path, fmt)


def _app_params(use_20k: bool) -> SpectrogramParams:
    """The app's "Use 20kHz" switch: stereo 10 Hz - 20 kHz, else mono 0 - 10 kHz."""
    if use_20k:
        return SpectrogramParams(min_frequency=10, max_frequency=20000, stereo=True)
    return SpectrogramParams(min_frequency=0, max_frequency=10000, stereo=False)


def _files_in(folder: str, pattern: str = "*", limit: int = -1) -> T.List[Path]:
    found = sorted(p for p in Path(folder).glob(pattern) if p.is_file())
    return found[:limit] if limit > 0 else found


def _try_load(path: Path):
    """Unreadable / non-audio files in a batch directory are skipped, as in the reference (cli.py:176-179, 247-250)."""
    try:
        return AudioSegment.from_file(str(path))
    except Exception:  # noqa: BLE001
        return None


def _run_pool(worker: T.Callable[[Path], None], items: T.Sequence[Path], num_threads: T.Optional[int]) -> None:
    with ThreadPool(processes=num_threads) as pool:
        for _ in pool.imap_unordered(worker, items):
            pass


# ------------------------------------------------------------------------------------------------ commands
def audio_to_image(*, audio: str, image: str, step_size_ms: int = 10, num_frequencies: int = 512,
                   min_frequency: int = 0, max_frequency: int = 10000, window_duration_ms: int = 100,
                   padded_duration_ms: int = 400, power_for_image: float = 0.25, stereo: bool = False,
                   device: str = "cuda"):
    """Compute a spectrogram image from a waveform."""
    clip = AudioSegment.from_file(audio)
    spec = SpectrogramParams(sample_rate=clip.frame_rate, stereo=stereo, step_size_ms=step_size_ms,
                             window_duration_ms=window_duration_ms, padded_duration_ms=padded_duration_ms,
                             num_frequencies=num_frequencies, min_frequency=min_frequency, max_frequency=max_frequency,
                             power_for_image=power_for_image)
    picture = SpectrogramImageConverter(params=spec, device=device).spectrogram_image_from_audio(clip)
    _store_image(picture, image, "PNG")
    print(f"Wrote {image}")


def print_exif(*, image: str) -> None:
    """Print the params of a spectrogram image as saved in the exif data."""
    for tag, value in image_util.exif_from_image(Image.open(image)).items():
        print(f"{tag:<20} = {value:>15}")


def image_to_audio(*, image: str, audio: str, device: str = "cuda"):
    """Reconstruct an audio clip from a spectrogram image."""
    picture = Image.open(image)
    tags = picture.getexif()
    assert tags is not None
    try:
        spec = SpectrogramParams.from_exif(exif=tags)
    except KeyError:       # an image without our tags: the reference falls back to the defaults with this message
        print("WARNING: Could not find spectrogram parameters in exif data. Using defaults.")
        spec = SpectrogramParams()
    clip = SpectrogramImageConverter(params=spec, device=device).audio_from_spectrogram_image(picture)
    clip.export(audio, format=Path(audio).suffix[1:])
    print(f"Wrote {audio} ({clip.duration_seconds:.2f} seconds)")


def sample_clips(*, audio: str, output_dir: str, num_clips: int = 1, duration_ms: int = 5120, mono: bool = False,
                 extension: str = "wav", seed: int = -1):
    """Slice an audio file into clips of the given duration."""
    if seed >= 0:
        np.random.seed(seed)
    source = AudioSegment.from_file(audio)
    if mono:
        source = source.set_channels(1)
    target = Path(output_dir)
    target.mkdir(parents=True, exist_ok=True)
    total_ms = int(source.duration_seconds * 1000)
    for index in range(num_clips):
        begin = np.random.randint(0, total_ms - duration_ms)
        out_path = target / f"clip_{index}_start_{begin}_ms_duration_{duration_ms}_ms.{extension}"
        source[begin: begin + duration_ms].export(out_path, format=extension)
        print(f"Wrote {out_path}")


def audio_to_images_batch(*, audio_dir: str, output_dir: str, image_extension: str = "jpg", step_size_ms: int = 10,
                          num_frequencies: int = 512, min_frequency: int = 0, max_frequency: int = 10000,
                          power_for_image: float = 0.25, mono: bool = False, sample_rate: int = 44100,
                          device: str = "cuda", num_threads: T.Optional[int] = None, limit: int = -1):
    """Process audio clips into spectrograms in batch, multi-threaded (one converter shared by all threads)."""
    target = Path(output_dir)
    target.mkdir(parents=True, exist_ok=True)
    spec = SpectrogramParams(sample_rate=sample_rate, stereo=not mono, step_size_ms=step_size_ms,
                             num_frequencies=num_frequencies, min_frequency=min_frequency, max_frequency=max_frequency,
                             power_for_image=power_for_image)
    shared = SpectrogramImageConverter(params=spec, device=device)
    want_channels = 1 if mono else 2

    def convert_one(path: Path) -> None:
        clip = _try_load(path)
        if clip is None:
            return
        if clip.channels != want_channels:
            clip = clip.set_channels(want_channels)
        if clip.frame_rate != spec.sample_rate:
            clip = clip.set_frame_rate(spec.sample_rate)
        _store_image(shared.spectrogram_image_from_audio(clip), target / f"{path.stem}.{image_extension}",
                     _PIL_FORMAT[image_extension])

    _run_pool(convert_one, _files_in(audio_dir, limit=limit), num_threads)


def sample_clips_batch(*, audio_dir: str, output_dir: str, num_clips_per_file: int = 1, duration_ms: int = 5120,
                       mono: bool = False, extension: str = "mp3", num_threads: T.Optional[int] = None, glob: str = "*",
                       limit: int = -1, seed: int = -1):
    """Sample short clips from a directory of audio files, multi-threaded."""
    sources = [p for p in _files_in(audio_dir, pattern=glob) if p.suffix != ".json"]      # metadata files never count (:219-220)
    if limit > 0:
        sources = sources[:limit]
    if seed >= 0:
        random.seed(seed)
    target = Path(output_dir)
    target.mkdir(parents=True, exist_ok=True)

    def cut_one(path: Path) -> None:
        source = _try_load(path)
        if source is None:
            return
        if mono:
            source = source.set_channels(1)
        total_ms = int(source.duration_seconds * 1000)
        for index in range(num_clips_per_file):
            try:        # a source no longer than the clip duration yields nothing, as in the reference (:247-250)
                begin = int(np.random.randint(0, total_ms - duration_ms))
            except ValueError:
                continue
            name = f"{path.stem}_{index}_start_{begin}_ms_dur_{duration_ms}_ms.{extension}"
            source[begin: begin + duration_ms].export(target / name, format=extension)

    _run_pool(cut_one, sources, num_threads)


def text_to_audio(*, prompt: str, audio: str, image: str = "", negative_prompt: str = "", seed: int = 42,
                  num_clips: int = 1, num_inference_steps: int = 30, guidance: float = 7.0, width: int = 512,
                  scheduler: str = "DPMSolverMultistepScheduler", use_20k: bool = False, loop: bool = False,
                  checkpoint: str = "riffusion/riffusion-model-v1", device: str = "cuda"):
    """Generate audio from a text prompt (Stable Diffusion txt2img, then spectrogram image -> audio); with --loop, a
    seamless loop."""
    from riffusion.riffusion_pipeline import RiffusionPipeline
    from riffusion.util import audio_util

    params = _app_params(use_20k)
    pipe = RiffusionPipeline.load_checkpoint(checkpoint=checkpoint, device=device)
    out = pipe.text_to_audio(prompt, params=params, negative_prompt=negative_prompt or None, seed=seed,
                             num_clips=num_clips, num_inference_steps=num_inference_steps, guidance_scale=guidance,
                             width=width, scheduler=scheduler, **(dict(loop=True) if loop else {}))
    images, waves = out["images"].cpu().numpy(), out["waveform"].cpu().numpy()

    def target(path: str, i: int) -> Path:
        p = Path(path)
        return p if num_clips == 1 else p.with_name(f"{p.stem}_{seed + i}{p.suffix}")

    for i in range(num_clips):
        segment = audio_util.apply_filters(
            audio_util.audio_from_waveform(samples=waves[i], sample_rate=params.sample_rate, normalize=True),
            compression=False)
        wav_path = target(audio, i)
        segment.export(str(wav_path), format=wav_path.suffix[1:])
        print(f"Wrote {wav_path} ({segment.duration_seconds:.2f} seconds)")
        if image:
            img_path = target(image, i)
            _store_spectrogram(images[i], params, img_path, _PIL_FORMAT.get(img_path.suffix[1:].lower(), "PNG"))
            print(f"Wrote {img_path}")


def parse_prompt_changes(prompt: str, changes: str) -> T.Union[str, T.List[T.Tuple[float, str]]]:
    """--prompt and --prompt-changes "20:jazz with drums;40:hard rock" -> [(0, prompt), (20, ...), (40, ...)], or the
    prompt alone without changes.  ValueError for an entry that is not <seconds>:<prompt>."""
    if not changes.strip():
        return prompt
    spans: T.List[T.Tuple[float, str]] = [(0.0, prompt)]
    for entry in changes.split(";"):
        start, sep, text = entry.partition(":")
        try:
            at = float(start) if sep else float("nan")
        except ValueError:
            at = float("nan")
        if not sep or at != at or not text.strip():
            raise ValueError(f"--prompt-changes entry {entry!r} is not <seconds>:<prompt>")
        spans.append((at, text.strip()))
    return spans


def text_to_track(*, prompt: str, audio: str, image: str = "", prompt_changes: str = "", negative_prompt: str = "",
                  duration_s: float = 30.0, seed: int = 42, num_tracks: int = 1, num_inference_steps: int = 30,
                  guidance: float = 7.0, scheduler: str = "DPMSolverMultistepScheduler", window_width: int = 512,
                  stride: int = 256, max_batch: int = 32, use_20k: bool = False,
                  checkpoint: str = "riffusion/riffusion-model-v1", device: str = "cuda"):
    """Generate a long track from text: overlapping clip windows denoised as one canvas (--window-width, --stride);
    --prompt-changes "20:jazz with drums;40:hard rock" switches the prompt at those times (seconds)."""
    from riffusion.riffusion_pipeline import RiffusionPipeline
    from riffusion.util import audio_util

    params = _app_params(use_20k)
    spans = parse_prompt_changes(prompt, prompt_changes)
    RiffusionPipeline.track_geometry(duration_s, window_width, stride, params.hop_length, params.sample_rate)
    RiffusionPipeline.track_prompts(spans, 1, window_width, stride, params.hop_length, params.sample_rate)
    pipe = RiffusionPipeline.load_checkpoint(checkpoint=checkpoint, device=device)
    out = pipe.text_to_track(spans, duration_s=duration_s, params=params, window_width=window_width, stride=stride,
                             negative_prompt=negative_prompt or None, seed=seed, num_tracks=num_tracks,
                             num_inference_steps=num_inference_steps, guidance_scale=guidance, scheduler=scheduler,
                             max_batch=max_batch)
    images, waves = out["images"].cpu().numpy(), out["waveform"].cpu().numpy()

    def target(path: str, i: int) -> Path:
        p = Path(path)
        return p if num_tracks == 1 else p.with_name(f"{p.stem}_{seed + i}{p.suffix}")

    for i in range(num_tracks):
        segment = audio_util.apply_filters(
            audio_util.audio_from_waveform(samples=waves[i], sample_rate=params.sample_rate, normalize=True),
            compression=False)
        wav_path = target(audio, i)
        segment.export(str(wav_path), format=wav_path.suffix[1:])
        print(f"Wrote {wav_path} ({segment.duration_seconds:.2f} seconds, {len(out['windows'])} windows)")
        if image:
            img_path = target(image, i)
            _store_spectrogram(images[i], params, img_path, _PIL_FORMAT.get(img_path.suffix[1:].lower(), "PNG"))
            print(f"Wrote {img_path}")


def audio_to_audio(*, audio: str, output: str, prompt: str, image_dir: str = "", negative_prompt: str = "",
                   seed: int = 42, denoising: float = 0.55, num_inference_steps: int = 25, guidance: float = 7.0,
                   scheduler: str = "DPMSolverMultistepScheduler", start_time_s: float = 0.0, duration_s: float = 20.0,
                   clip_duration_s: float = 5.0, overlap_duration_s: float = 0.2, prompt_b: str = "", seed_b: int = -1,
                   denoising_b: float = -1.0, max_batch: int = 32, use_20k: bool = False, magic_mix: bool = False,
                   kmin: float = 0.3, kmax: float = 0.5, mix_factor: float = 0.5,
                   checkpoint: str = "riffusion/riffusion-model-v1", device: str = "cuda"):
    """Riff a track with a text prompt (overlapping clips, img2img, crossfaded back together); with --prompt-b,
    interpolate from --prompt to --prompt-b along the track (--seed-b / --denoising-b: -1 = same as the first end);
    with --magic-mix, restyle each clip with Magic Mix, keeping its layout (--kmin, --kmax, --mix-factor)."""
    from riffusion.riffusion_pipeline import RiffusionPipeline

    params = _app_params(use_20k)
    track = AudioSegment.from_file(audio)
    pipe = RiffusionPipeline.load_checkpoint(checkpoint=checkpoint, device=device)
    out = pipe.audio_to_audio(
        track, prompt, params=params, start_time_s=start_time_s, duration_s=duration_s, clip_duration_s=clip_duration_s,
        overlap_duration_s=overlap_duration_s, negative_prompt=negative_prompt or None, seed=seed, denoising=denoising,
        num_inference_steps=num_inference_steps, guidance_scale=guidance, scheduler=scheduler,
        prompt_b=prompt_b or None, seed_b=None if seed_b < 0 else seed_b,
        denoising_b=None if denoising_b < 0 else denoising_b, max_batch=max_batch, magic_mix=magic_mix, kmin=kmin,
        kmax=kmax, mix_factor=mix_factor)
    segment = out["segment"]
    segment.export(output, format=Path(output).suffix[1:])
    print(f"Wrote {output} ({segment.duration_seconds:.2f} seconds, {len(out['clip_start_times'])} clips)")
    if image_dir:
        target = Path(image_dir)
        target.mkdir(parents=True, exist_ok=True)
        for kind in ("source", "riffed"):
            images = out["source_images" if kind == "source" else "images"].cpu().numpy()
            for i, im in enumerate(images):
                _store_spectrogram(im, params, target / f"clip_{i}_{kind}.png")
        print(f"Wrote {2 * len(images)} images to {image_dir}")


def interpolation(*, prompt_a: str, prompt_b: str, seed_image: str, output: str, image_dir: str = "", seed_a: int = 42,
                  seed_b: int = 42, denoising_a: float = 0.75, denoising_b: float = 0.75, guidance: float = 7.0,
                  num_interpolation_steps: int = 12, num_inference_steps: int = 50, alpha_power: float = 1.0,
                  max_batch: int = 32, checkpoint: str = "riffusion/riffusion-model-v1", device: str = "cuda"):
    """Walk from --prompt-a (--seed-a, --denoising-a) to --prompt-b (--seed-b, --denoising-b) on a seed spectrogram
    image in --num-interpolation-steps clips, appended into one track (--alpha-power shapes the walk)."""
    from riffusion.datatypes import PromptInput
    from riffusion.riffusion_pipeline import DEFAULT_PARAMS, RiffusionPipeline

    start = PromptInput(prompt=prompt_a, seed=seed_a, denoising=denoising_a, guidance=guidance)
    end = PromptInput(prompt=prompt_b, seed=seed_b, denoising=denoising_b, guidance=guidance)
    init_image = Image.open(seed_image).convert("RGB")
    pipe = RiffusionPipeline.load_checkpoint(checkpoint=checkpoint, device=device)
    out = pipe.interpolation(start, end, init_image, num_interpolation_steps=num_interpolation_steps,
                             num_inference_steps=num_inference_steps, alpha_power=alpha_power, max_batch=max_batch)
    segment = out["segment"]
    segment.export(output, format=Path(output).suffix[1:])
    print(f"Wrote {output} ({segment.duration_seconds:.2f} seconds, {len(out['alphas'])} steps)")
    if image_dir:
        target = Path(image_dir)
        target.mkdir(parents=True, exist_ok=True)
        for i, im in enumerate(out["images"].cpu().numpy()):
            _store_spectrogram(im, DEFAULT_PARAMS, target / f"step_{i}.png")
        print(f"Wrote {len(out['alphas'])} images to {image_dir}")


def text_to_audio_batch(*, json: str, output_dir: str, num_seeds: int = 1, max_batch: int = 32,
                        audio_extension: str = "wav", checkpoint: str = "riffusion/riffusion-model-v1",
                        device: str = "cuda"):
    """Generate audio for every (entry, seed, param set) of a JSON file of param sets and prompts (the app's Text to
    Audio Batch format), writing image_*.jpg / audio_* per clip and index.json to --output-dir."""
    import json as json_module

    from riffusion.riffusion_pipeline import DEFAULT_PARAMS, RiffusionPipeline
    from riffusion.text_to_audio_batch import build_index, output_names, parse_batch, plan_batch

    data = json_module.loads(Path(json).read_text())
    param_sets, entries = parse_batch(data)
    clips, _ = plan_batch(param_sets, entries, num_seeds, max_batch)      # refuses bad counts before loading weights
    for ps in param_sets:
        if ps.checkpoint != checkpoint:
            print(f"{ps.name}: names checkpoint {ps.checkpoint!r}; every clip runs on {checkpoint!r}")
    pipe = RiffusionPipeline.load_checkpoint(checkpoint=checkpoint, device=device)
    out = pipe.text_to_audio_batch(data, num_seeds=num_seeds, max_batch=max_batch)
    target = Path(output_dir)
    target.mkdir(parents=True, exist_ok=True)
    paths = []
    for clip, res in zip(clips, out["clips"]):
        image_name, audio_name = output_names(clip.param_index, entries[clip.entry_index], clip.seed, audio_extension)
        _store_spectrogram(res["image"].cpu().numpy(), DEFAULT_PARAMS, target / image_name, "JPEG")
        res["segment"].export(str(target / audio_name), format=audio_extension)
        paths.append((str(target / image_name), str(target / audio_name)))
    (target / "index.json").write_text(json_module.dumps(build_index(data, param_sets, clips, paths), indent=4))
    print(f"Wrote {len(clips)} clips in {len(out['loops'])} loops and index.json to {output_dir}")


COMMANDS = [audio_to_image, image_to_audio, sample_clips, print_exif, audio_to_images_batch, sample_clips_batch]
# commands of this package that the reference's CLI does not have; `main` offers them next to COMMANDS
EXTRA_COMMANDS = [text_to_audio]
# the track-level commands, offered by `main` after EXTRA_COMMANDS
TRACK_COMMANDS = [audio_to_audio, interpolation, text_to_track]
# the file-driven batch commands, offered by `main` after TRACK_COMMANDS
BATCH_COMMANDS = [text_to_audio_batch]


# ------------------------------------------------------------------------------------------------ argparse front end
def _str2bool(v: str) -> bool:
    if v.lower() in ("1", "true", "yes", "y"):
        return True
    if v.lower() in ("0", "false", "no", "n"):
        return False
    raise argparse.ArgumentTypeError(f"expected a boolean, got {v!r}")


def build_parser(commands: T.Sequence[T.Callable] = tuple(COMMANDS)) -> argparse.ArgumentParser:
    """argh-style front end: one sub-command per function (underscores -> dashes), one --flag per keyword-only arg.
    By default the reference's six commands exactly; `main` passes COMMANDS + EXTRA_COMMANDS."""
    parser = argparse.ArgumentParser(prog="riffusion.cli", description=__doc__)
    sub = parser.add_subparsers(dest="command", required=True)
    for fn in commands:
        sp = sub.add_parser(fn.__name__.replace("_", "-"), help=(fn.__doc__ or "").strip())
        sp.set_defaults(_fn=fn)
        for name, prm in inspect.signature(fn).parameters.items():
            flag = "--" + name.replace("_", "-")
            if prm.default is inspect.Parameter.empty:
                sp.add_argument(flag, dest=name, required=True)
            elif isinstance(prm.default, bool):
                sp.add_argument(flag, dest=name, nargs="?", const=True, default=prm.default, type=_str2bool)
            elif prm.default is None:
                sp.add_argument(flag, dest=name, default=None, type=int)
            else:
                sp.add_argument(flag, dest=name, default=prm.default, type=type(prm.default))
    return parser


def main(argv: T.Optional[T.Sequence[str]] = None) -> None:
    args = vars(build_parser(COMMANDS + EXTRA_COMMANDS + TRACK_COMMANDS + BATCH_COMMANDS).parse_args(argv))
    fn = args.pop("_fn")
    args.pop("command")
    fn(**args)


if __name__ == "__main__":
    main(sys.argv[1:])
