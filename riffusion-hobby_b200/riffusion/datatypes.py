"""Request / response schema of the inference API.

Field names, order and defaults are those of the reference's riffusion/datatypes.py:10-73 (the Flask server fills them
from request JSON with `dacite`; that package is not on the GPU image, so `from_dict` below does the same nested
construction for the two input types, rejecting unknown keys like dacite's strict mode).
"""
from __future__ import annotations

import dataclasses
import typing as T
from dataclasses import dataclass


def _build(cls, payload: T.Mapping[str, T.Any]):
    known = {f.name for f in dataclasses.fields(cls)}
    extra = set(payload) - known
    if extra:
        raise KeyError(f"{cls.__name__}: unknown field(s) {sorted(extra)}")
    return cls(**payload)


@dataclass(frozen=True)
class PromptInput:
    """One end point of an interpolation.

    prompt           text that conditions the denoiser
    seed             seeds the noise tensor of this end point (and, for `start`, the VAE posterior draw)
    negative_prompt  carried in the schema; `RiffusionPipeline.riffuse` never forwards it (a quirk kept from the reference)
    denoising        img2img strength in (0, 1]: 0.75 keeps the seed image's structure, 1.0 ignores it
    guidance         classifier-free guidance scale
    """

    prompt: str
    seed: int
    negative_prompt: T.Optional[str] = None
    denoising: float = 0.75
    guidance: float = 7.0

    @classmethod
    def from_dict(cls, payload: T.Mapping[str, T.Any]) -> "PromptInput":
        return _build(cls, payload)


@dataclass(frozen=True)
class InferenceInput:
    """A (start, end, alpha) interpolation request on a seed spectrogram image: alpha = 0 reproduces `start`, alpha = 1
    `end`; prompts are interpolated linearly in embedding space, the noise tensors spherically."""

    start: PromptInput
    end: PromptInput
    alpha: float
    num_inference_steps: int = 50
    seed_image_id: str = "og_beat"
    mask_image_id: T.Optional[str] = None

    @classmethod
    def from_dict(cls, payload: T.Mapping[str, T.Any]) -> "InferenceInput":
        fields = dict(payload)
        for side in ("start", "end"):
            if isinstance(fields.get(side), T.Mapping):
                fields[side] = PromptInput.from_dict(fields[side])
        return _build(cls, fields)


@dataclass(frozen=True)
class InferenceOutput:
    """What the model server answers with: the generated spectrogram (base64 JPEG), its audio (base64 MP3) and the clip
    length in seconds."""

    image: str
    audio: str
    duration_s: float
