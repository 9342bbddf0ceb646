"""Host-side bookkeeping of the app's Text to Audio Batch task (riffusion/streamlit/tasks/text_to_audio_batch.py): the
JSON file of parameter sets and prompt entries, the order the app renders clips in, the batched loops they are grouped
into, the output file names and `index.json`.  `RiffusionPipeline.text_to_audio_batch` runs the loops on the device;
the `text-to-audio-batch` command writes the files.

A valid input (the app's own example has a trailing comma that `json.loads` rejects):

    {
      "params": [
        {"name": "g5", "scheduler": "DPMSolverMultistepScheduler", "num_inference_steps": 50, "guidance": 5.0},
        {"name": "g7", "scheduler": "DPMSolverMultistepScheduler", "num_inference_steps": 50, "guidance": 7.0}
      ],
      "entries": [
        {"prompt": "Church bells", "seed": 42},
        {"prompt": "electronic beats", "negative_prompt": "drums", "seed": 100},
        {"prompt": "classical violin concerto", "seed": 4}
      ]
    }

`params` is one parameter set or a list of them; a set's missing keys take the app's defaults (`PARAM_DEFAULTS`) and a
set without a name is called "params[i]".  An entry's `seed` defaults to 42.  Unlike the app, an unknown key is refused
instead of ignored, so a misspelt "guidance_scale" cannot silently run at guidance 7.0.  The keys the app and the
command write back (`image_path`, `audio_path`, `outputs`) are accepted, so an `index.json` can be fed back in.
"""
from __future__ import annotations

import copy
import dataclasses
import typing as T

from riffusion.scheduler_b200 import SCHEDULERS, make_scheduler

PARAM_DEFAULTS = dict(checkpoint="riffusion/riffusion-model-v1", scheduler="DPMSolverMultistepScheduler",
                      num_inference_steps=50, guidance=7.0, width=512)
PARAM_KEYS = {"name", *PARAM_DEFAULTS}
ENTRY_KEYS = {"prompt", "negative_prompt", "seed", "image_path", "audio_path", "outputs"}
TOP_KEYS = {"params", "entries"}


@dataclasses.dataclass(frozen=True)
class ParamSet:
    name: str
    checkpoint: str
    scheduler: str
    num_inference_steps: int
    guidance: float
    width: int


@dataclasses.dataclass(frozen=True)
class Entry:
    prompt: str
    negative_prompt: T.Optional[str]
    seed: int


@dataclasses.dataclass(frozen=True)
class Clip:
    """One generated clip: param set `param_index` applied to entry `entry_index` at `seed`."""
    param_index: int
    entry_index: int
    seed: int


@dataclasses.dataclass(frozen=True)
class Loop:
    """One batched CFG loop: the clips `rows` (indices into the clip list) share scheduler, steps, width and the side
    of guidance 1; `n_unet_evals` CFG UNet evaluations."""
    scheduler: str
    num_inference_steps: int
    width: int
    cfg: bool
    rows: T.Tuple[int, ...]
    n_unet_evals: int


def _unknown(obj: dict, allowed: T.Set[str], where: str) -> None:
    extra = sorted(set(obj) - allowed)
    if extra:
        raise ValueError(f"unknown key(s) {', '.join(map(repr, extra))} in {where}; allowed: {', '.join(sorted(allowed))}")


def _int(value, what: str) -> int:
    if isinstance(value, bool) or not isinstance(value, int):
        raise ValueError(f"{what} must be an integer, got {value!r}")
    return value


def parse_batch(data: T.Any) -> T.Tuple[T.List[ParamSet], T.List[Entry]]:
    """The parameter sets and entries of a loaded batch JSON object, with the app's defaults filled in.  Raises
    ValueError for a missing `params` or `entries`, no entries, an entry without a prompt, a width that is not a positive
    multiple of 64, fewer than 1 step, a scheduler other than DPM-Solver++, PNDM, DDIM and Euler ancestral, or an unknown
    key."""
    if not isinstance(data, dict):
        raise ValueError(f"the batch must be a JSON object, got {type(data).__name__}")
    for key in ("params", "entries"):
        if key not in data:
            raise ValueError(f"the batch has no {key!r}")
    _unknown(data, TOP_KEYS, "the batch")
    raw_params = data["params"] if isinstance(data["params"], list) else [data["params"]]
    if not raw_params:
        raise ValueError("the batch has no parameter set")
    param_sets = []
    for i, p in enumerate(raw_params):
        where = f"params[{i}]"
        if not isinstance(p, dict):
            raise ValueError(f"{where} must be an object, got {p!r}")
        _unknown(p, PARAM_KEYS, where)
        full = {**PARAM_DEFAULTS, "name": where, **p}
        steps = _int(full["num_inference_steps"], f"{where}.num_inference_steps")
        width = _int(full["width"], f"{where}.width")
        if steps < 1:
            raise ValueError(f"{where}.num_inference_steps must be at least 1, got {steps}")
        if width <= 0 or width % 64:
            raise ValueError(f"{where}.width must be a positive multiple of 64, got {width}")
        if full["scheduler"] not in SCHEDULERS:
            raise ValueError(f"unsupported scheduler {full['scheduler']!r} in {where}; supported: {', '.join(SCHEDULERS)}")
        if isinstance(full["guidance"], bool) or not isinstance(full["guidance"], (int, float)):
            raise ValueError(f"{where}.guidance must be a number, got {full['guidance']!r}")
        param_sets.append(ParamSet(name=str(full["name"]), checkpoint=str(full["checkpoint"]),
                                   scheduler=full["scheduler"], num_inference_steps=steps,
                                   guidance=float(full["guidance"]), width=width))
    if not isinstance(data["entries"], list) or not data["entries"]:
        raise ValueError("the batch's 'entries' must be a non-empty list")
    entries = []
    for i, e in enumerate(data["entries"]):
        where = f"entries[{i}]"
        if not isinstance(e, dict):
            raise ValueError(f"{where} must be an object, got {e!r}")
        _unknown(e, ENTRY_KEYS, where)
        if not isinstance(e.get("prompt"), str):
            raise ValueError(f"{where} has no prompt")
        neg = e.get("negative_prompt")
        if neg is not None and not isinstance(neg, str):
            raise ValueError(f"{where}.negative_prompt must be a string, got {neg!r}")
        entries.append(Entry(prompt=e["prompt"], negative_prompt=neg, seed=_int(e.get("seed", 42), f"{where}.seed")))
    return param_sets, entries


def n_unet_evals(scheduler: str, num_inference_steps: int) -> int:
    """CFG evaluations of one txt2img loop: one per timestep (n for DPM-Solver++, DDIM and Euler ancestral, n + 1 for
    PNDM)."""
    sched = make_scheduler(scheduler)
    sched.set_timesteps(num_inference_steps)
    return len(sched.timesteps)


def plan_batch(param_sets: T.Sequence[ParamSet], entries: T.Sequence[Entry], num_seeds: int = 1,
               max_batch: int = 32) -> T.Tuple[T.List[Clip], T.List[Loop]]:
    """The clips in the app's order (entry, then seed entry.seed .. entry.seed + num_seeds - 1, then param set) and the
    loops that run them: clips grouped by (scheduler, steps, width, guidance > 1) in order of first appearance, each
    group cut into chunks of at most `max_batch` rows in clip order.  Sets that differ only in guidance (on one side of
    1) share a loop; each row keeps its own guidance."""
    if num_seeds < 1:
        raise ValueError(f"num_seeds must be at least 1, got {num_seeds}")
    if max_batch < 1:
        raise ValueError(f"max_batch must be at least 1, got {max_batch}")
    clips = [Clip(param_index=p, entry_index=e, seed=seed)
             for e, entry in enumerate(entries)
             for seed in range(entry.seed, entry.seed + num_seeds)
             for p in range(len(param_sets))]
    groups: T.Dict[T.Tuple[str, int, int, bool], T.List[int]] = {}
    for i, clip in enumerate(clips):
        ps = param_sets[clip.param_index]
        groups.setdefault((ps.scheduler, ps.num_inference_steps, ps.width, ps.guidance > 1.0), []).append(i)
    loops = []
    for (scheduler, steps, width, cfg), rows in groups.items():
        evals = n_unet_evals(scheduler, steps)
        for lo in range(0, len(rows), max_batch):
            loops.append(Loop(scheduler=scheduler, num_inference_steps=steps, width=width, cfg=cfg,
                              rows=tuple(rows[lo:lo + max_batch]), n_unet_evals=evals))
    return clips, loops


def output_names(param_index: int, entry: Entry, seed: int, audio_extension: str) -> T.Tuple[str, str]:
    """(image, audio) file names of a clip: the app's image_{i}_{prompt}_neg_{negative}.jpg / audio_... with spaces
    turned into underscores, plus _{seed}.  The app's names have no seed, so with several seeds all but the last are
    overwritten there."""
    stem = f"{param_index}_{entry.prompt.replace(' ', '_')}_neg_{(entry.negative_prompt or '').replace(' ', '_')}_{seed}"
    return f"image_{stem}.jpg", f"audio_{stem}.{audio_extension}"


def build_index(data: dict, param_sets: T.Sequence[ParamSet], clips: T.Sequence[Clip],
                paths: T.Sequence[T.Tuple[str, str]]) -> dict:
    """`index.json`: the input with each param set's name filled in, and per entry the app's `image_path` /
    `audio_path` (the last clip written for it, as in the app) and an `outputs` list of {name, seed, image_path,
    audio_path} for every clip of the entry.  paths[k] = (image path, audio path) of clips[k]."""
    index = copy.deepcopy(data)
    if isinstance(index["params"], list):
        for p, ps in zip(index["params"], param_sets):
            p["name"] = ps.name
    else:
        index["params"]["name"] = param_sets[0].name
    for e in index["entries"]:
        e["outputs"] = []
    for clip, (image_path, audio_path) in zip(clips, paths):
        e = index["entries"][clip.entry_index]
        e["image_path"], e["audio_path"] = image_path, audio_path
        e["outputs"].append(dict(name=param_sets[clip.param_index].name, seed=clip.seed, image_path=image_path,
                                 audio_path=audio_path))
    return index
