"""RiffusionPipeline — H100-native drop-in for riffusion/riffusion_pipeline.py.

Same public surface as the reference class (`load_checkpoint`, `riffuse`, `interpolate_img2img`, `embed_text`,
`embed_text_weighted`, `device`, module-level `preprocess_image` / `preprocess_mask`) and the same control flow
around the inner seams (`self.unet(...)`, `self.scheduler.*`, `self.vae.*`), but those seams are the wgmma
implementations of this package (UNetB200, PNDMSchedulerB200, VaeB200) instead of diffusers modules.

What is NOT here: diffusers (`DiffusionPipeline.from_pretrained`, hub download, traced-UNet download) — none of
it is installable in this image.  Checkpoints are loaded from diffusers-format state dicts on disk
(`load_checkpoint` on a local directory holding `unet/`, `vae/` weights as .safetensors/.bin), or created with
random-init SD-1.5 weights (`random_init`, BASELINE config 4).  The CLIP text encoder is outside the hot path
(runs once per prompt, lru-cached in the reference); it is used through `transformers` when a tokenizer / text
encoder is supplied, otherwise callers pass text embeddings directly.
"""
from __future__ import annotations

import functools
import math
import typing as T
from pathlib import Path

import numpy as np
import torch
from PIL import Image

from riffusion import tc_ops as ops
from riffusion import window_ops
from riffusion.datatypes import InferenceInput
from riffusion.scheduler_b200 import (DDIMSchedulerB200, EulerAncestralSchedulerB200, PNDMSchedulerB200,
                                      make_scheduler)
from riffusion.spectrogram_params import SpectrogramParams
from riffusion.unet_b200 import UNetB200
from riffusion.util import torch_util
from riffusion.vae_b200 import VaeB200, _Posterior

VAE_SCALE = 0.18215
# the spectrogram parameters of text_to_audio / audio_to_audio when none are given: the app's mono 0-10 kHz
DEFAULT_PARAMS = SpectrogramParams(min_frequency=0, max_frequency=10000, stereo=False)


class RiffusionPipeline:
    """Prompt / seed interpolation on spectrogram images (img2img), running on one H100."""

    def __init__(self, vae: VaeB200, unet: UNetB200, scheduler: T.Optional[PNDMSchedulerB200] = None,
                 text_encoder=None, tokenizer=None, device: str = "cuda"):
        self.vae, self.unet = vae, unet
        self.scheduler = scheduler or PNDMSchedulerB200()
        self.text_encoder, self.tokenizer = text_encoder, tokenizer
        self._device = torch.device(device)
        self._moment_cache: T.Dict[int, T.Tuple[torch.Tensor, torch.Tensor]] = {}
        self.device_slerp = True        # rf_slerp_f16 instead of the reference's host-numpy round trip
        self.use_cuda_graph = True      # replay each CFG UNet evaluation as one CUDA graph
        self._graphs: T.Dict[T.Tuple, T.Any] = {}

    # ------------------------------------------------------------------------------ construction
    @classmethod
    def random_init(cls, seed: int = 0, device: str = "cuda", with_vae: bool = True) -> "RiffusionPipeline":
        """Random-init SD-1.5 architecture (N(0, 0.02^2) weights), BASELINE config 4 — there is no network to
        fetch riffusion/riffusion-model-v1."""
        from riffusion.sd15_spec import random_state_dicts

        unet_sd, vae_sd = random_state_dicts(seed, with_vae=with_vae)
        vae = VaeB200(vae_sd, device=device) if with_vae else None
        return cls(vae=vae, unet=UNetB200(unet_sd, device=device), device=device)

    @classmethod
    def load_checkpoint(cls, checkpoint: str, use_traced_unet: bool = True, channels_last: bool = False,
                        dtype: torch.dtype = torch.float16, device: str = "cuda", local_files_only: bool = False,
                        low_cpu_mem_usage: bool = False, cache_dir: T.Optional[str] = None) -> "RiffusionPipeline":
        """Load a diffusers-layout checkpoint directory (`unet/diffusion_pytorch_model.{safetensors,bin}`,
        `vae/...`, optional `text_encoder/`, `tokenizer/`).  Signature kept from riffusion_pipeline.py:63-125;
        `use_traced_unet` / `channels_last` are accepted and ignored (the wgmma UNet already is the fast path,
        activations are always channels-last)."""
        device = torch_util.check_device(device)
        if dtype != torch.float16:
            raise ValueError("the H100-native pipeline computes in fp16 (the reference forces fp32 only on CPU/MPS)")
        root = Path(checkpoint)
        if not root.is_dir():
            raise FileNotFoundError(
                f"{checkpoint!r} is not a local diffusers checkpoint directory; hub download is not available "
                "(no diffusers / network in this build)")
        unet_sd = _load_weights(root / "unet")
        vae_sd = _load_weights(root / "vae")
        text_encoder = tokenizer = None
        if (root / "text_encoder").is_dir() and (root / "tokenizer").is_dir():
            from transformers import CLIPTextModel, CLIPTokenizer

            tokenizer = CLIPTokenizer.from_pretrained(root / "tokenizer")
            text_encoder = CLIPTextModel.from_pretrained(root / "text_encoder", torch_dtype=torch.float16).to(device)
        return cls(vae=VaeB200(vae_sd, device=device), unet=UNetB200(unet_sd, device=device),
                   text_encoder=text_encoder, tokenizer=tokenizer, device=device)

    @property
    def device(self) -> str:
        return str(self._device)

    # ------------------------------------------------------------------------------ text
    @functools.lru_cache()
    def embed_text(self, text) -> torch.Tensor:
        """CLIP embedding of a prompt, (1, 77, 768) fp16 (riffusion_pipeline.py:177-191)."""
        if self.tokenizer is None or self.text_encoder is None:
            raise RuntimeError("no text encoder loaded: pass text embeddings to interpolate_img2img directly")
        ids = self.tokenizer(text, padding="max_length", max_length=self.tokenizer.model_max_length, truncation=True,
                             return_tensors="pt").input_ids
        with torch.no_grad():
            return self.text_encoder(ids.to(self.device))[0].to(torch.float16)

    @functools.lru_cache()
    def embed_text_weighted(self, text) -> torch.Tensor:
        """CLIP embedding with "(word:1.2)" / "[word]" attention weights (riffusion_pipeline.py:193-206 ->
        external/prompt_weighting.py:236-372): parse, encode in chunks of 75 tokens, scale token rows by their weights,
        restore the mean."""
        from riffusion.external.prompt_weighting import get_weighted_text_embeddings

        if self.tokenizer is None or self.text_encoder is None:
            raise RuntimeError("no text encoder loaded: pass text embeddings to interpolate_img2img directly")
        with torch.no_grad():
            return get_weighted_text_embeddings(pipe=self, prompt=text, uncond_prompt=None, max_embeddings_multiples=3,
                                                no_boseos_middle=False, skip_parsing=False, skip_weighting=False)[0]

    # ------------------------------------------------------------------------------ riffuse
    @torch.no_grad()
    def riffuse(self, inputs: InferenceInput, init_image: Image.Image, mask_image: T.Optional[Image.Image] = None,
                use_reweighting: bool = True) -> Image.Image:
        """Interpolate between the two prompts / seeds of `inputs` on `init_image` (riffusion_pipeline.py:208-287)."""
        alpha = inputs.alpha
        start, end = inputs.start, inputs.end
        guidance_scale = start.guidance * (1.0 - alpha) + end.guidance * alpha
        generator_start = torch.Generator(device=self.device).manual_seed(start.seed)
        generator_end = torch.Generator(device=self.device).manual_seed(end.seed)
        embed = self.embed_text_weighted if use_reweighting else self.embed_text
        embed_start, embed_end = embed(start.prompt), embed(end.prompt)
        text_embedding = embed_start + alpha * (embed_end - embed_start)          # linear, not slerp (:249)

        init_latents = self.encode_image(init_image, torch.Generator(device=self.device).manual_seed(start.seed))
        mask = None
        if mask_image:
            vae_scale_factor = 2 ** (len(self.vae.config.block_out_channels) - 1)
            mask = preprocess_mask(mask_image, scale_factor=vae_scale_factor).to(device=self.device, dtype=embed_start.dtype)
        outputs = self.interpolate_img2img(
            text_embeddings=text_embedding, init_latents=init_latents, mask=mask, generator_a=generator_start,
            generator_b=generator_end, interpolate_alpha=alpha, strength_a=start.denoising, strength_b=end.denoising,
            num_inference_steps=inputs.num_inference_steps, guidance_scale=guidance_scale)
        return outputs["images"][0]

    @torch.no_grad()
    def riffuse_batch(self, inputs: T.Sequence[InferenceInput],
                      init_images: T.Union[None, Image.Image, T.Sequence[Image.Image]],
                      mask_image: T.Optional[Image.Image] = None, use_reweighting: bool = True, *,
                      moments: T.Optional[T.Tuple[torch.Tensor, torch.Tensor]] = None,
                      output_type: str = "pil") -> T.List[T.Any]:
        """`riffuse` for a list of requests in one batched denoising loop (SURVEY 8(f)-2) — what
        streamlit/tasks/interpolation.py:146-164 does one request at a time.  Every request draws exactly what `riffuse`
        draws for it (posterior noise and noise_a from generator(start.seed), noise_b from generator(end.seed), per-request
        alpha for the slerp and the prompt interpolation), so result i equals `riffuse(inputs[i], ...)` up to the batch-size
        dependent accumulation order of the kernels.  Requests are grouped by (strength, guidance, steps): the PNDM state
        and the guidance scalar are shared inside a group.

        `moments` = (mean, logvar), each (len(inputs), 4, h, w), replaces the VAE encoding of `init_images` (pass None
        for them): request i starts from row i.  `output_type="latent"` returns each request's (1, 4, h, w) latents
        (1/0.18215-scaled) instead of a PIL image."""
        if moments is None:
            images = [init_images] * len(inputs) if isinstance(init_images, Image.Image) else list(init_images)
            if len(images) != len(inputs):
                raise ValueError(f"{len(images)} init images for {len(inputs)} requests")
        elif init_images is not None or moments[0].shape[0] != len(inputs):
            raise ValueError(f"moments replace init_images (pass None for them) and need one row per request "
                             f"({len(inputs)}), got {moments[0].shape[0]}")
        embed = self.embed_text_weighted if use_reweighting else self.embed_text
        groups: T.Dict[T.Tuple, T.List[int]] = {}
        for i, inp in enumerate(inputs):
            a = inp.alpha
            strength = (1 - a) * inp.start.denoising + a * inp.end.denoising
            guidance = inp.start.guidance * (1.0 - a) + inp.end.guidance * a
            # exact floats, not rounded: `int(num_inference_steps * strength)` (:361) depends on the last bit of the
            # reference's own lerp (alpha 0.3, denoising 0.75 -> 0.7499999999999999 -> one evaluation fewer)
            groups.setdefault((strength, guidance, inp.num_inference_steps), []).append(i)
        mask = None
        if mask_image:
            vae_scale_factor = 2 ** (len(self.vae.config.block_out_channels) - 1)
            mask = preprocess_mask(mask_image, scale_factor=vae_scale_factor).to(device=self.device, dtype=torch.float16)
        results: T.List[T.Optional[Image.Image]] = [None] * len(inputs)
        for (strength, guidance, steps), idx in groups.items():
            texts, lats, noise = self._prepare_requests(inputs, idx, embed, images if moments is None else None, moments)
            out = self.interpolate_img2img(
                text_embeddings=texts, init_latents=lats, mask=mask, generator_a=None, generator_b=None,
                interpolate_alpha=0.0, strength_a=strength, strength_b=strength, num_inference_steps=steps,
                guidance_scale=guidance, noise=noise, output_type=output_type)
            for j, i in enumerate(idx):
                results[i] = out["latents"][j:j + 1] if output_type == "latent" else out["images"][j]
        return results  # type: ignore[return-value]

    def _prepare_requests(self, inputs: T.Sequence[InferenceInput], idx: T.Sequence[int], embed,
                          images: T.Optional[T.Sequence[Image.Image]],
                          moments: T.Optional[T.Tuple[torch.Tensor, torch.Tensor]]):
        """What `riffuse` draws for each request inputs[i], i in idx: the prompt embeddings lerped at the request's
        alpha, the VAE posterior sample of images[i] (or of row i of `moments`) and noise_a from a generator seeded with
        start.seed, noise_b from one seeded with end.seed, and their slerp at alpha.  Returns (text embeddings, latents,
        noise), one row per request in idx order."""
        texts, lats, nas, nbs, alphas = [], [], [], [], []
        for i in idx:
            inp = inputs[i]
            e0, e1 = embed(inp.start.prompt), embed(inp.end.prompt)
            texts.append(e0 + inp.alpha * (e1 - e0))
            g_post = torch.Generator(device=self.device).manual_seed(inp.start.seed)
            if moments is None:
                lats.append(self.encode_image(images[i], g_post))
            else:
                lats.append(_sample_latents(moments[0][i:i + 1], moments[1][i:i + 1], g_post))
            ga = torch.Generator(device=self.device).manual_seed(inp.start.seed)
            gb = torch.Generator(device=self.device).manual_seed(inp.end.seed)
            shape = lats[-1].shape
            nas.append(torch.randn(shape, generator=ga, device=self.device, dtype=torch.float16))
            nbs.append(torch.randn(shape, generator=gb, device=self.device, dtype=torch.float16))
            alphas.append(float(inp.alpha))
        na, nb = torch.cat(nas), torch.cat(nbs)
        if self.device_slerp:
            noise = ops.slerp(alphas, na, nb)
        else:
            noise = torch.cat([torch_util.slerp(al, na[j:j + 1], nb[j:j + 1]) for j, al in enumerate(alphas)])
        return torch.cat(texts), torch.cat(lats), noise

    # ------------------------------------------------------------------------------ interpolation
    @staticmethod
    def interpolation_alphas(n: int, p: float = 1.0) -> np.ndarray:
        """The alphas of the app's interpolation task (streamlit/tasks/interpolation.py:99-104): linspace(0, 1, n) mapped
        through x = 2a - 1, a' = (|x|^p sign(x) + 1) / 2, so p > 1 packs the alphas towards 0.5 and p < 1 towards the two ends."""
        a = np.linspace(0, 1, n) * 2 - 1
        return (np.abs(a) ** p * np.sign(a) + 1) / 2

    @torch.no_grad()
    def interpolation(self, start, end, init_image: Image.Image, *, num_interpolation_steps: int = 12,
                      num_inference_steps: int = 50, alpha_power: float = 1.0, params=None, max_batch: int = 32,
                      init_angles: T.Optional[torch.Tensor] = None, apply_filters: bool = True) -> T.Dict[str, T.Any]:
        """A track that walks from `start` to `end` (PromptInputs: prompt, seed, denoising, guidance) on `init_image`:
        the app's Interpolation task (streamlit/tasks/interpolation.py:99-181).  Clip i is `riffuse` of
        InferenceInput(alpha_i, num_inference_steps, start, end) with alpha_i = interpolation_alphas(n, alpha_power)[i]
        (PNDM, weighted prompts, no negative prompt, no mask), turned into audio with `params` (default mono 0-10 kHz)
        and appended to the previous clips without a crossfade.

        Every row draws what `riffuse` draws for its request (`_prepare_requests`) and is noised at its own start
        timestep; then up to `max_batch` rows run as one CFG loop (`PNDMRowsB200`): each row joins at its own
        `_img2img_steps` start and keeps its own guidance, so a walk whose ends differ in denoising or guidance still
        runs as one loop.  After the loop, on the device: VAE decode -> uint8 image -> mel -> waveform
        (`init_angles` (n, channels, n_fft/2 + 1, frames) fixes Griffin-Lim's initial phases); on the host:
        peak-normalised int16, `apply_filters`, `stitch_segments` with no crossfade.  The page round-trips each clip
        through MP3 bytes before joining; here the clips are joined as int16 PCM.

        Raises ValueError before any device work when num_interpolation_steps or max_batch is below 1, when the two
        ends' guidance lies on different sides of 1, or when the seed image's height (rounded down to a multiple of 32)
        is not params.num_frequencies.  Returns dict(segment, images ((n, H, W, 3) uint8 device
        tensor), waveform ((n, channels, L) fp32 before normalisation), alphas, requests, n_unet_evals (per loop))."""
        from riffusion.util import audio_util

        n = num_interpolation_steps
        if n < 1:
            raise ValueError("num_interpolation_steps must be at least 1")
        if max_batch < 1:
            raise ValueError("max_batch must be at least 1")
        if (start.guidance > 1.0) != (end.guidance > 1.0):
            raise ValueError(f"the guidance of the two ends ({start.guidance}, {end.guidance}) lies on different sides "
                             "of 1: only some clips would use classifier-free guidance")
        params = DEFAULT_PARAMS if params is None else params
        if init_image.height - init_image.height % 32 != params.num_frequencies:
            raise ValueError(f"the seed image is {init_image.height} pixels high; params.num_frequencies "
                             f"{params.num_frequencies} needs that height (rounded down to a multiple of 32)")
        alphas = self.interpolation_alphas(n, alpha_power)
        requests = [InferenceInput(start=start, end=end, alpha=float(a), num_inference_steps=num_inference_steps)
                    for a in alphas]
        sched = PNDMSchedulerB200()
        sched.set_timesteps(num_inference_steps)
        strengths = [(1 - r.alpha) * start.denoising + r.alpha * end.denoising for r in requests]   # as riffuse
        guidances = [start.guidance * (1.0 - r.alpha) + end.guidance * r.alpha for r in requests]
        steps = [self._img2img_steps(sched, num_inference_steps, s) for s in strengths]
        converter = self._converter(params, None)
        images = [init_image] * n
        u8s, waves, n_evals = [], [], []
        for lo in range(0, n, max_batch):
            idx = list(range(lo, min(n, lo + max_batch)))
            angles = None if init_angles is None else init_angles[lo:lo + len(idx)]
            u8, wave, evals = self._rows_loop(requests, idx, images, sched, [steps[i] for i in idx],
                                              [guidances[i] for i in idx], converter, params.stereo, angles)
            n_evals.append(evals)
            waves.append(wave)
            u8s.append(u8)
        waveform = torch.cat(waves)
        segments = []
        for w in waveform.cpu().numpy():
            seg = audio_util.audio_from_waveform(samples=w, sample_rate=params.sample_rate, normalize=True)
            segments.append(audio_util.apply_filters(seg, compression=False) if apply_filters else seg)
        return dict(segment=audio_util.stitch_segments(segments, crossfade_s=0), images=torch.cat(u8s),
                    waveform=waveform, alphas=alphas, requests=requests, n_unet_evals=n_evals)

    def _rows_loop(self, requests: T.Sequence[InferenceInput], idx: T.Sequence[int],
                   images: T.Sequence[Image.Image], sched, starts: T.Sequence[T.Tuple[int, int]],
                   guidances: T.Sequence[float], converter, stereo: bool, angles: T.Optional[torch.Tensor], *,
                   masks: T.Optional[T.Sequence[T.Optional[torch.Tensor]]] = None,
                   n_fill: int = 0, waveform: bool = True) -> T.Tuple[torch.Tensor, T.Optional[torch.Tensor], int]:
        """The loop body of `interpolation` and `riffuse_requests`: requests[i], i in idx, as the rows of one CFG loop.
        Row k draws what `riffuse` draws for its request (`_prepare_requests`), is noised at
        sched.timesteps[-init_timestep] with (init_timestep, t_start) = starts[k], and joins a `PNDMRowsB200` loop of
        type(sched) at its own t_start with guidances[k].  masks[k], a (1, 4, h, w) fp16 device mask or None, gives row k
        riffuse's inpainting blend inside the step kernel.  `n_fill` filler rows, copies of the last row that start at
        len(timesteps) and so never step, pad the loop's batch; they are dropped before the VAE.  After the loop, on the
        device: VAE decode -> uint8 image -> waveform (`angles` fixes Griffin-Lim's initial phases; None with
        `waveform=False`).  Returns (uint8 images, waveform, UNet evaluations)."""
        from riffusion.scheduler_b200 import PNDMRowsB200

        texts, lats, noise = self._prepare_requests(requests, idx, self.embed_text_weighted, images, None)
        lats = lats.to(device=self._device, dtype=torch.float16).contiguous()
        noise = noise.to(self._device, torch.float16).contiguous()
        latents = torch.cat([sched.add_noise(lats[k:k + 1], noise[k:k + 1], int(sched.timesteps[-starts[k][0]]))
                             for k in range(len(idx))])
        if n_fill:
            def pad(t: torch.Tensor) -> torch.Tensor:
                return torch.cat([t, t[-1:].expand(n_fill, *t.shape[1:])]).contiguous()

            texts, lats, noise, latents = pad(texts), pad(lats), pad(noise), pad(latents)
        masks = [None] * len(idx) if masks is None else list(masks)
        t_starts = [s[1] for s in starts] + [len(sched.timesteps)] * n_fill
        rows = PNDMRowsB200(sched.num_inference_steps, t_starts, list(guidances) + [guidances[-1]] * n_fill,
                            device=self._device, scheduler=type(sched),
                            masked=[m is not None for m in masks] + [False] * n_fill)
        if rows.masked:
            blank = torch.zeros_like(lats[:1])
            mask = torch.cat([blank if m is None else m.to(device=self._device, dtype=torch.float16).expand_as(blank)
                              for m in masks] + [blank] * n_fill).contiguous()
            rows.set_mask_inputs(init=lats, noise=noise, mask=mask)
        context = self._context(None, None, len(t_starts), guidances[0] > 1.0, texts, None)
        latents, evals = self._denoise(rows, rows.timesteps, latents, context, guidances[0])
        u8 = self._decode_u8((1.0 / VAE_SCALE) * latents[:len(idx)])
        wave = self._u8_to_waveform(u8, converter, stereo, angles) if waveform else None
        return u8, wave, evals

    def context_error(self, inputs: InferenceInput) -> T.Optional[str]:
        """Why `riffuse` cannot build this request's CFG context, or None.  Its weighted prompts embed to 77 k tokens:
        the start and end embeddings must have one length for the lerp, and with guidance above 1 that length must be
        the unconditional embedding's (77).  `riffuse` (as the reference) fails inside torch otherwise."""
        e0 = self.embed_text_weighted(inputs.start.prompt)
        e1 = self.embed_text_weighted(inputs.end.prompt)
        if e0.shape != e1.shape:
            return f"the start and end prompts embed to {e0.shape[1]} and {e1.shape[1]} tokens"
        guidance = inputs.start.guidance * (1.0 - inputs.alpha) + inputs.end.guidance * inputs.alpha
        n_uncond = self.embed_text("").shape[1]
        if guidance > 1.0 and e0.shape[1] != n_uncond:
            return (f"the prompts embed to {e0.shape[1]} tokens; guidance {guidance} needs {n_uncond}, the length of the "
                    "unconditional embedding")
        return None

    @staticmethod
    def request_loops(keys: T.Sequence[T.Hashable], max_batch: int) -> T.List[T.Tuple[T.List[int], int]]:
        """The loops of `riffuse_requests` for requests with these group keys: one group per distinct key, in order of
        first arrival, requests in arrival order, cut into chunks of at most `max_batch`.  Each chunk runs at a batch of
        its row count rounded up to a power of two, at most `max_batch`, so a pipeline captures at most
        log2(max_batch) + 2 CUDA graphs per (latent shape, context shape).  Returns [(request indices, batch)]."""
        if max_batch < 1:
            raise ValueError("max_batch must be at least 1")
        groups: T.Dict[T.Hashable, T.List[int]] = {}
        for i, key in enumerate(keys):
            groups.setdefault(key, []).append(i)
        loops = []
        for idx in groups.values():
            for lo in range(0, len(idx), max_batch):
                chunk = idx[lo:lo + max_batch]
                loops.append((chunk, min(max_batch, 1 << (len(chunk) - 1).bit_length())))
        return loops

    @torch.no_grad()
    def riffuse_requests(self, inputs: T.Sequence[InferenceInput], init_images: T.Sequence[Image.Image],
                         mask_images: T.Sequence[T.Optional[Image.Image]], *, max_batch: int = 16,
                         init_angles: T.Optional[T.Sequence[torch.Tensor]] = None,
                         waveform: bool = True) -> T.List[T.Dict[str, T.Any]]:
        """`riffuse` of many requests, each with its own seed image and optional mask, in as few CFG loops as their
        shapes allow: the model server's batch entry point.

        One loop per group of (num_inference_steps, latent shape, context length, guidance > 1), requests in arrival
        order, chunked at `max_batch` (`request_loops`).  In its loop each request is a row that draws what `riffuse`
        draws for it, joins at its own `_img2img_steps` start with its own lerped guidance and, with a mask, applies
        riffuse's inpainting blend after each of its steps (`PNDMRowsB200` with `masked`).  A chunk's batch is its row
        count rounded up to a power of two (at most `max_batch`); the filler rows never step and are dropped.  After
        each loop, on the device: VAE decode -> uint8 image -> mel -> waveform, mono 0-10 kHz; `init_angles`, one
        (1, n_fft/2 + 1, frames) complex64 tensor per request, fixes Griffin-Lim's initial phases; `waveform=False`
        skips the audio (the results' waveform is None).  The pipeline's scheduler must be PNDM or DDIM.

        Raises ValueError before any device work for another scheduler, lists of other lengths, max_batch below 1, or
        a mask whose size differs from its seed image, and before any loop for prompts whose context `riffuse` cannot
        build (`context_error`), naming the request.  Returns per request dict(image ((H, W, 3) uint8 device tensor),
        waveform ((1, L) fp32 before normalisation), loop (the loop's index), n_unet_evals (its loop's), filler_rows
        (its loop's))."""
        n = len(inputs)
        if type(self.scheduler) not in (PNDMSchedulerB200, DDIMSchedulerB200):
            raise ValueError(f"riffuse_requests runs PNDM or DDIM rows, not {type(self.scheduler).__name__}")
        if len(init_images) != n or len(mask_images) != n or (init_angles is not None and len(init_angles) != n):
            raise ValueError(f"need one seed image, one mask (or None) and one set of angles per request: {n} requests, "
                             f"{len(init_images)} images, {len(mask_images)} masks")
        if max_batch < 1:
            raise ValueError("max_batch must be at least 1")
        for i, (img, mask) in enumerate(zip(init_images, mask_images)):
            if mask is not None and mask.size != img.size:
                raise ValueError(f"request {i}: mask image is {mask.size[0]}x{mask.size[1]}, its seed image "
                                 f"{img.size[0]}x{img.size[1]}")
        for i, r in enumerate(inputs):
            error = self.context_error(r)
            if error is not None:
                raise ValueError(f"request {i}: {error}")
        sched_cls = type(self.scheduler)
        strengths = [(1 - r.alpha) * r.start.denoising + r.alpha * r.end.denoising for r in inputs]    # as riffuse
        guidances = [r.start.guidance * (1.0 - r.alpha) + r.end.guidance * r.alpha for r in inputs]
        keys = []
        for r, img, g in zip(inputs, init_images, guidances):
            w, h = img.size
            ctx = self.embed_text_weighted(r.start.prompt).shape[1]
            keys.append((r.num_inference_steps, ((h - h % 32) // 8, (w - w % 32) // 8), ctx, g > 1.0))
        scale = 2 ** (len(self.vae.config.block_out_channels) - 1)
        masks = [None if m is None else preprocess_mask(m, scale_factor=scale).to(device=self.device, dtype=torch.float16)
                 for m in mask_images]
        converter = self._converter(DEFAULT_PARAMS, None) if waveform else None
        results: T.List[T.Optional[T.Dict[str, T.Any]]] = [None] * n
        for loop, (idx, batch) in enumerate(self.request_loops(keys, max_batch)):
            sched = sched_cls()
            sched.set_timesteps(inputs[idx[0]].num_inference_steps)
            starts = [self._img2img_steps(sched, sched.num_inference_steps, strengths[i]) for i in idx]
            angles = None if init_angles is None else torch.stack([init_angles[i] for i in idx])
            u8, wave, evals = self._rows_loop(inputs, idx, init_images, sched, starts, [guidances[i] for i in idx],
                                              converter, DEFAULT_PARAMS.stereo, angles,
                                              masks=[masks[i] for i in idx], n_fill=batch - len(idx),
                                              waveform=waveform)
            for k, i in enumerate(idx):
                results[i] = dict(image=u8[k], waveform=None if wave is None else wave[k], loop=loop, n_unet_evals=evals,
                                  filler_rows=batch - len(idx))
        return results  # type: ignore[return-value]

    def encode_image(self, init_image: Image.Image, generator: torch.Generator) -> torch.Tensor:
        """preprocess + VAE posterior sample * 0.18215 (:252-264).  The (mean, logvar) moments only depend on the
        image and are cached; the posterior noise is drawn from `generator` like the reference."""
        key = hash(init_image.tobytes()) ^ hash(init_image.size)
        if key not in self._moment_cache:
            img = preprocess_image(init_image).to(device=self.device, dtype=torch.float16)
            self._moment_cache[key] = self.vae.encode_moments(img)
        mean, logvar = self._moment_cache[key]
        return _sample_latents(mean, logvar, generator)

    @staticmethod
    def img2img_start(scheduler, num_inference_steps: int, strength: float) -> int:
        """Index of the first timestep an img2img loop runs, `t_start`; `img2img` adds noise at timesteps[t_start] and
        runs timesteps[t_start:].  The rule of `interpolate_img2img`, see `_img2img_steps`.  For DPM-Solver++ this
        restates diffusers' img2img pipeline from memory and is not pinned against diffusers (unpinned)."""
        return RiffusionPipeline._img2img_steps(scheduler, num_inference_steps, strength)[1]

    @staticmethod
    def _img2img_steps(scheduler, num_inference_steps: int, strength: float) -> T.Tuple[int, int]:
        """(init_timestep, t_start) of `interpolate_img2img` (riffusion_pipeline.py:358-392):
        init_timestep = min(int(steps * strength) + offset, steps), t_start = max(steps - init_timestep + offset, 0),
        offset = the scheduler's step offset (1 for PNDM, 0 for DPM-Solver++).  `interpolate_img2img` adds noise at
        timesteps[-init_timestep], which is timesteps[t_start] whenever the loop runs at least one step."""
        offset = scheduler.config.get("steps_offset", 0)
        init_timestep = min(int(num_inference_steps * strength) + offset, num_inference_steps)
        return init_timestep, max(num_inference_steps - init_timestep + offset, 0)

    # ------------------------------------------------------------------------------ denoising loop
    @torch.no_grad()
    def interpolate_img2img(self, text_embeddings: torch.Tensor, init_latents: torch.Tensor,
                            generator_a: torch.Generator, generator_b: torch.Generator, interpolate_alpha: float,
                            mask: T.Optional[torch.Tensor] = None, strength_a: float = 0.8, strength_b: float = 0.8,
                            num_inference_steps: int = 50, guidance_scale: float = 7.5,
                            negative_prompt: T.Optional[T.Union[str, T.List[str]]] = None,
                            num_images_per_prompt: int = 1, eta: T.Optional[float] = 0.0,
                            output_type: T.Optional[str] = "pil", uncond_embeddings: T.Optional[torch.Tensor] = None,
                            noise_a: T.Optional[torch.Tensor] = None, noise_b: T.Optional[torch.Tensor] = None,
                            noise: T.Optional[torch.Tensor] = None, **kwargs) -> T.Dict[str, T.Any]:
        """riffusion_pipeline.py:289-436.  Extra keyword-only inputs (`uncond_embeddings`, `noise_a`, `noise_b`)
        let callers inject what the reference computes internally (CLIP("") and the generator draws) — used by
        the parity tests and by runs without a text encoder.  The pipeline's scheduler may be PNDM (eta is ignored, as
        the reference's PNDM ignores it) or DDIM (eta must be 0; ValueError otherwise)."""
        batch_size = text_embeddings.shape[0]
        sched = self.scheduler
        if isinstance(sched, EulerAncestralSchedulerB200):
            raise ValueError("interpolate_img2img runs PNDM or DDIM; Euler ancestral needs per-step noise (use img2img)")
        if eta and isinstance(sched, DDIMSchedulerB200):
            raise ValueError(f"DDIM runs with eta = 0 only, got eta {eta}")
        sched.set_timesteps(num_inference_steps)
        dev = self._device
        text_embeddings = text_embeddings.to(device=dev, dtype=torch.float16)
        bs_embed, seq_len, _ = text_embeddings.shape
        text_embeddings = text_embeddings.repeat(1, num_images_per_prompt, 1).view(bs_embed * num_images_per_prompt, seq_len, -1)

        do_cfg = guidance_scale > 1.0
        if do_cfg:
            if uncond_embeddings is None:
                if negative_prompt is None:                                    # :328-335
                    uncond_tokens = [""]
                elif isinstance(negative_prompt, str):
                    uncond_tokens = [negative_prompt]
                elif batch_size != len(negative_prompt):
                    raise ValueError("The length of `negative_prompt` should be equal to batch_size.")
                else:
                    uncond_tokens = list(negative_prompt)
                if self.tokenizer is None:
                    raise RuntimeError("classifier-free guidance needs the CLIP embedding of ''; pass uncond_embeddings")
                ids = self.tokenizer(uncond_tokens, padding="max_length", max_length=self.tokenizer.model_max_length,
                                     truncation=True, return_tensors="pt").input_ids
                uncond_embeddings = self.text_encoder(ids.to(self.device))[0]
            if num_images_per_prompt > 1 and uncond_embeddings.shape[0] == batch_size:
                # one row per prompt, repeated like the text rows above (:347-350)
                uncond_embeddings = uncond_embeddings.repeat_interleave(num_images_per_prompt, dim=0)
        context = self._context(None, None, batch_size * num_images_per_prompt, do_cfg, text_embeddings,
                                uncond_embeddings)                                                 # :354

        latents_dtype = torch.float16
        strength = (1 - interpolate_alpha) * strength_a + interpolate_alpha * strength_b          # :358
        init_timestep, t_start = self._img2img_steps(sched, num_inference_steps, strength)        # :361-363, :392
        t_noise = int(sched.timesteps[-init_timestep])                                            # :365
        init_latents = init_latents.to(device=dev, dtype=latents_dtype).contiguous()
        if noise is None:
            if noise_a is None:
                noise_a = torch.randn(init_latents.shape, generator=generator_a, device=self.device, dtype=latents_dtype)
            if noise_b is None:
                noise_b = torch.randn(init_latents.shape, generator=generator_b, device=self.device, dtype=latents_dtype)
            if self.device_slerp:      # fp32 reductions on the GPU, no device->host->device round trip
                noise = ops.slerp(interpolate_alpha, noise_a.to(dev, latents_dtype), noise_b.to(dev, latents_dtype))
            else:                      # the reference's host-numpy slerp in fp16 (bit-compatible)
                noise = torch_util.slerp(interpolate_alpha, noise_a.to(dev, latents_dtype), noise_b.to(dev, latents_dtype))
        noise = noise.to(dev, latents_dtype).contiguous()
        latents = sched.add_noise(init_latents, noise, t_noise)                                    # :379
        latents, n_evals = self._denoise(sched, sched.timesteps[t_start:], latents, context, guidance_scale,
                                         mask=mask, init=init_latents, noise=noise)                # :398-425
        # :427-436 — "latents" is the 1/0.18215-scaled tensor, as the reference returns it
        out = self._finish(latents, n_evals, output_type)
        out["nsfw_content_detected"] = False
        return out

    def _graphed_unet(self, latent_shape, context: torch.Tensor, wrap_w: bool = False):
        """The CUDA-graph CFG evaluation for this (latent shape, context shape, wrap_w), or None when graphs are off."""
        if not self.use_cuda_graph:
            return None
        from riffusion.graphed import GraphedUNet

        # one captured graph per (latent shape, context shape, loop mode); a new request only refreshes the
        # cross-attention K / V^T that the graph reads (capture costs two eager evaluations + instantiation).  Loop and
        # non-loop evaluations run different convolutions, so they never share a graph.
        gkey = (tuple(latent_shape), tuple(context.shape)) + (("wrap_w",) if wrap_w else ())
        graphed = self._graphs.get(gkey)
        if graphed is None:
            graphed = self._graphs[gkey] = (GraphedUNet(self.unet, latent_shape, context, wrap_w=True) if wrap_w else
                                            GraphedUNet(self.unet, latent_shape, context))
        else:
            graphed.set_context(context)
        return graphed

    # ------------------------------------------------------------------------------ text -> image
    @torch.no_grad()
    def txt2img(self, prompt: str, *, negative_prompt: T.Optional[str] = None, seed: int = 42, num_clips: int = 1,
                num_inference_steps: int = 30, guidance_scale: float = 7.0, width: int = 512, height: int = 512,
                scheduler: str = "DPMSolverMultistepScheduler", output_type: T.Optional[str] = "pil",
                text_embeddings: T.Optional[torch.Tensor] = None, uncond_embeddings: T.Optional[torch.Tensor] = None,
                latents: T.Optional[torch.Tensor] = None,
                step_noise: T.Optional[torch.Tensor] = None, loop: bool = False) -> T.Dict[str, T.Any]:
        """Text to spectrogram image: Stable Diffusion txt2img, the reference app's text-to-audio generation.

        Clip i starts from `torch.randn((1, 4, height/8, width/8))` drawn from a CUDA generator seeded with `seed + i`
        (one pipeline call per seed in the app), times the scheduler's `init_noise_sigma`; all clips run as one CFG
        batch.  The prompt and the negative prompt (default "") are encoded without prompt weighting.  `scheduler` is
        "DPMSolverMultistepScheduler", "PNDMScheduler", "DDIMScheduler" or "EulerAncestralDiscreteScheduler"; a fresh
        instance is used per call.  Euler ancestral also draws one fp16 tensor per step from each clip's generator,
        after its latents (`_step_noise`).  `width` and `height` must be multiples of 64 (diffusers accepts multiples of
        8).  `text_embeddings` / `uncond_embeddings` / `latents` / `step_noise` (steps, clips, 4, h, w) replace the text
        encoder and the generator draws.  `loop`: every 3x3 convolution of the UNet and of the VAE decoder pads circularly
        along the width, so the image tiles horizontally (a seamless loop).  Returns dict(images, latents
        (1/0.18215-scaled), latents_unscaled, n_unet_evals)."""
        if width <= 0 or height <= 0 or width % 64 or height % 64:
            raise ValueError(f"width and height must be positive multiples of 64, got {width}x{height}")
        if num_clips < 1:
            raise ValueError("num_clips must be at least 1")
        sched = make_scheduler(scheduler)
        sched.set_timesteps(num_inference_steps)
        dev = self._device
        context = self._context(prompt, negative_prompt, num_clips, guidance_scale > 1.0, text_embeddings,
                                uncond_embeddings)
        shape = (1, 4, height // 8, width // 8)
        gens = [torch.Generator(device=self.device).manual_seed(seed + i) for i in range(num_clips)]
        if latents is None:
            latents = torch.cat([torch.randn(shape, generator=g, device=self.device, dtype=torch.float16) for g in gens])
        latents = latents.to(device=dev, dtype=torch.float16).contiguous()
        if tuple(latents.shape) != (num_clips,) + shape[1:]:
            raise ValueError(f"latents must be {(num_clips,) + shape[1:]}, got {tuple(latents.shape)}")
        self._step_noise(sched, len(sched.timesteps), latents, step_noise, gens)
        if sched.init_noise_sigma != 1.0:
            latents = (latents * sched.init_noise_sigma).contiguous()
        if loop:        # the default call stays exactly what it was
            latents, n_evals = self._denoise(sched, sched.timesteps, latents, context, guidance_scale, wrap_w=True)
            return self._finish(latents, n_evals, output_type, wrap_w=True)
        latents, n_evals = self._denoise(sched, sched.timesteps, latents, context, guidance_scale)
        return self._finish(latents, n_evals, output_type)

    def _context(self, prompt: str, negative_prompt: T.Optional[str], n: int, do_cfg: bool,
                 text_embeddings: T.Optional[torch.Tensor], uncond_embeddings: T.Optional[torch.Tensor]) -> torch.Tensor:
        """[uncond | text] for n clips (text only without guidance): plain `embed_text` of the prompt and of the negative
        prompt (default ""), or the injected embeddings (1 or n rows each)."""
        dev = self._device

        def rows(emb: torch.Tensor, name: str) -> torch.Tensor:
            emb = emb.to(device=dev, dtype=torch.float16)
            emb = emb.expand(n, -1, -1) if emb.shape[0] == 1 else emb
            if emb.shape[0] != n:
                raise ValueError(f"{name} hold {emb.shape[0]} rows for {n} clips")
            return emb

        text = rows(self.embed_text(prompt) if text_embeddings is None else text_embeddings, "text_embeddings")
        if not do_cfg:
            return text.contiguous()
        uncond = self.embed_text(negative_prompt or "") if uncond_embeddings is None else uncond_embeddings
        return torch.cat([rows(uncond, "uncond_embeddings"), text]).contiguous()

    def _step_noise(self, sched, n_steps: int, latents: torch.Tensor, step_noise: T.Optional[torch.Tensor],
                    generators: T.Sequence[torch.Generator]) -> None:
        """Hand an Euler-ancestral scheduler the z of each of the loop's `n_steps` steps, (n_steps, B, ...) fp16:
        `step_noise` when given, else n_steps draws of torch.randn((1, ...), fp16) per row from that row's generator,
        continuing its stream, as diffusers' step draws them from the pipeline's generator.  One generator for B rows
        means the rows' streams are identical (img2img seeds every image alike) and its draws serve every row.  Other
        schedulers draw nothing and take no step_noise (ValueError)."""
        if not isinstance(sched, EulerAncestralSchedulerB200):
            if step_noise is not None:
                raise ValueError("step_noise is only used by EulerAncestralDiscreteScheduler")
            return
        want = (n_steps,) + tuple(latents.shape)
        if step_noise is None:
            row = (1,) + tuple(latents.shape[1:])
            draws = [torch.cat([torch.randn(row, generator=g, device=self.device, dtype=torch.float16)
                                for _ in range(n_steps)]) if n_steps else latents.new_empty((0,) + row[1:])
                     for g in generators]
            step_noise = torch.stack(draws, dim=1) if len(draws) > 1 else draws[0][:, None].expand(want)
        step_noise = step_noise.to(device=latents.device, dtype=torch.float16).contiguous()
        if tuple(step_noise.shape) != want:
            raise ValueError(f"step_noise must be {want}, got {tuple(step_noise.shape)}")
        sched.set_step_noise(step_noise)

    def _denoise(self, sched, timesteps, latents: torch.Tensor, context: torch.Tensor, guidance_scale: float,
                 mask: T.Optional[torch.Tensor] = None, init: T.Optional[torch.Tensor] = None,
                 noise: T.Optional[torch.Tensor] = None,
                 layout: T.Optional[T.Tuple[float, torch.Tensor, torch.Tensor, int]] = None,
                 wrap_w: bool = False, windows: T.Optional[window_ops.Windows] = None) -> T.Tuple[torch.Tensor, int]:
        """The CFG loop over `timesteps`: one UNet evaluation of [latents | latents] (a captured CUDA graph when enabled)
        and one fused guidance + scheduler step each.  With a `mask`, every step is followed by the inpainting blend of
        interpolate_img2img (:420-425): `init` noised with `noise` at that step's timestep where the mask is 1, the
        stepped latents where it is 0.  With `layout` = (mix_factor, enc, noise32, stop), steps 1 .. stop - 1 of the
        loop are Magic Mix's layout phase: the UNet evaluates mix_factor * latents + (1 - mix_factor) * add_noise(enc,
        noise32, t) (`tc_ops.magic_mix`) and the scheduler still steps the latents.  The UNet input passes through
        `sched.scale_model_input` (the identity, without a launch, for every scheduler but Euler ancestral).  The UNet,
        the graph and the scheduler receive the scheduler's own timestep values: ints, or floats for Euler ancestral.
        `wrap_w`: the UNet pads circularly along W (seamless loops).  `windows` (long tracks): `latents` is a canvas of
        `windows.canvas` columns; each step gathers its windows (`window_ops.window_gather`), evaluates the UNet on them
        (context: one row per window, track-major) and merges both halves of the eps pair back onto the canvas
        (`window_ops.window_merge`) before the scheduler steps the canvas.  Returns (latents, evaluations)."""
        do_cfg = guidance_scale > 1.0
        ctx_cache: T.Dict[str, T.Any] = {}
        graphed = None
        unet_shape = latents.shape
        if windows is not None:
            unet_shape = (latents.shape[0] * windows.n,) + tuple(latents.shape[1:3]) + (windows.width,)
        if do_cfg:
            graphed = self._graphed_unet(unet_shape, context, True) if wrap_w else self._graphed_unet(unet_shape, context)
        loop_kw = dict(wrap_w=True) if wrap_w else {}
        if mask is not None:
            mask = mask.to(device=latents.device, dtype=latents.dtype).expand_as(latents).contiguous()
        n_evals = 0
        for j, t in enumerate(timesteps):
            t_val = t.item() if torch.is_tensor(t) else t
            unet_in = latents
            if layout is not None and 0 < j < layout[3]:
                a = float(sched.alphas_cumprod[t_val])
                unet_in = ops.magic_mix(latents, layout[1], layout[2], a ** 0.5, (1.0 - a) ** 0.5, layout[0])
            unet_in = sched.scale_model_input(unet_in, t_val)
            if windows is not None:
                unet_in = window_ops.window_gather(unet_in, windows)
            if graphed is not None:
                eps_pair = graphed(unet_in, t_val)
            else:
                model_in = torch.cat([unet_in] * 2) if do_cfg else unet_in
                eps_pair = self.unet(model_in, t_val, encoder_hidden_states=context, ctx_cache=ctx_cache, **loop_kw).sample
            if windows is not None:
                eps_pair = window_ops.window_merge(eps_pair, windows)
            n_evals += 1
            if not do_cfg:
                eps_pair = torch.cat([eps_pair, eps_pair])
            latents = sched.step_cfg(eps_pair, guidance_scale if do_cfg else 0.0, t_val, latents)
            if mask is not None:
                latents = sched.add_noise(init, noise, t_val, mask=mask, blend_with=latents)
        return latents, n_evals

    def _finish(self, latents: torch.Tensor, n_evals: int, output_type: T.Optional[str],
                wrap_w: bool = False) -> T.Dict[str, T.Any]:
        """dict(latents (1/0.18215-scaled), latents_unscaled, n_unet_evals, images): PIL images, a float16 (B, H, W, 3)
        array in [0, 1] for any other output_type, or None for "latent" and without a VAE.  `wrap_w`: the decoder pads
        circularly along W."""
        scaled = (1.0 / VAE_SCALE) * latents
        out: T.Dict[str, T.Any] = dict(latents=scaled, latents_unscaled=latents, n_unet_evals=n_evals)
        if output_type == "latent" or self.vae is None:
            out["images"] = None
        elif output_type == "pil":
            u8 = self._decode_u8(scaled, True) if wrap_w else self._decode_u8(scaled)
            out["images"] = [Image.fromarray(im) for im in u8.cpu().numpy()]
        else:
            image = (self.vae.decode(scaled, wrap_w=True) if wrap_w else self.vae.decode(scaled)).sample
            out["images"] = (image / 2 + 0.5).clamp(0, 1).cpu().permute(0, 2, 3, 1).numpy()
        return out

    def _decode_u8(self, scaled_latents: torch.Tensor, wrap_w: bool = False) -> torch.Tensor:
        """VAE decode -> (B, H, W, 3) uint8 images: `(image / 2 + 0.5).clamp(0, 1)` -> numpy_to_pil (:430-434) in the fp16
        arithmetic of the reference's CUDA path, on the device.  `wrap_w`: the decoder pads circularly along W."""
        if wrap_w:
            return ops.vae_image_to_u8(self.vae.decode(scaled_latents, wrap_w=True).sample)
        return ops.vae_image_to_u8(self.vae.decode(scaled_latents).sample)

    # ------------------------------------------------------------------------------ image -> image
    @torch.no_grad()
    def img2img(self, prompt: str, images: T.Union[torch.Tensor, T.Sequence[Image.Image]], *, strength: float = 0.55,
                num_inference_steps: int = 25, guidance_scale: float = 7.0, negative_prompt: T.Optional[str] = None,
                seed: int = 42, scheduler: str = "DPMSolverMultistepScheduler", output_type: T.Optional[str] = "pil",
                text_embeddings: T.Optional[torch.Tensor] = None, uncond_embeddings: T.Optional[torch.Tensor] = None,
                noise: T.Optional[torch.Tensor] = None,
                moments: T.Optional[T.Tuple[torch.Tensor, torch.Tensor]] = None,
                step_noise: T.Optional[torch.Tensor] = None) -> T.Dict[str, T.Any]:
        """Image to image: diffusers' StableDiffusionImg2ImgPipeline as the reference app calls it
        (streamlit/util.py:354-396), for a batch of images in one CFG loop.

        `images`: PIL images (preprocessed like `preprocess_image`) or a (B, 3, H, W) fp16 device tensor in [-1, 1]; H and
        W must be multiples of 64.  Image i is denoised with its own generator seeded with `seed` (the app uses one seed
        for every clip), which draws the VAE posterior noise (fp32) first and then the img2img noise (fp16).  The start
        point follows `img2img_start` (unpinned for DPM-Solver++, DDIM and Euler ancestral): noise is added at
        timesteps[t_start], then timesteps[t_start:] are run.  `scheduler`: "DPMSolverMultistepScheduler",
        "PNDMScheduler", "DDIMScheduler" or "EulerAncestralDiscreteScheduler", a fresh instance per call; Euler ancestral
        then draws one fp16 tensor per step run from the same generator, after the img2img noise, and since every image's
        generator has drawn the same shapes from the same seed, one stream serves all images.  `text_embeddings` /
        `uncond_embeddings` / `noise` (B, 4, H/8, W/8) / `step_noise` (steps run, B, 4, H/8, W/8) replace the text
        encoder and the generator draws; `moments` = (mean, logvar) replaces the VAE encoding of `images` (pass None for
        them).
        Returns dict(images, latents (1/0.18215-scaled), latents_unscaled, n_unet_evals, t_start)."""
        sched = make_scheduler(scheduler)
        sched.set_timesteps(num_inference_steps)
        dev = self._device
        mean, logvar = self._image_moments(images, moments)
        n = mean.shape[0]
        context = self._context(prompt, negative_prompt, n, guidance_scale > 1.0, text_embeddings, uncond_embeddings)
        lats, draws = [], []
        for i in range(n):
            g = torch.Generator(device=self.device).manual_seed(seed)
            lats.append(_sample_latents(mean[i:i + 1], logvar[i:i + 1], g))
            draws.append(torch.randn(lats[-1].shape, generator=g, device=self.device, dtype=torch.float16))
        stream = g                          # the state every image's generator is in now
        init_latents = torch.cat(lats).to(device=dev, dtype=torch.float16).contiguous()
        noise = torch.cat(draws) if noise is None else noise.to(device=dev, dtype=torch.float16)
        if noise.shape != init_latents.shape:
            raise ValueError(f"noise must be {tuple(init_latents.shape)}, got {tuple(noise.shape)}")
        t_start = self.img2img_start(sched, num_inference_steps, strength)
        timesteps = sched.timesteps[t_start:]
        self._step_noise(sched, len(timesteps), init_latents, step_noise, [stream])
        latents = init_latents
        if len(timesteps):
            latents = sched.add_noise(init_latents, noise, timesteps[0].item())
        latents, n_evals = self._denoise(sched, timesteps, latents, context, guidance_scale)
        out = self._finish(latents, n_evals, output_type)
        out["t_start"] = t_start
        return out

    def _image_moments(self, images, moments: T.Optional[T.Tuple[torch.Tensor, torch.Tensor]]):
        """`moments` when given, else the VAE (mean, logvar) of `images`: PIL images (preprocessed like
        `preprocess_image`) or a (B, 3, H, W) fp16 tensor in [-1, 1], H and W multiples of 64."""
        if moments is not None:
            return moments
        if not torch.is_tensor(images):
            images = torch.cat([preprocess_image(im) for im in images])
        images = images.to(device=self._device, dtype=torch.float16)
        if images.dim() != 4 or images.shape[1] != 3 or images.shape[2] % 64 or images.shape[3] % 64:
            raise ValueError(f"images must be (B, 3, H, W) with H and W multiples of 64, got {tuple(images.shape)}")
        return self.vae.encode_moments(images.contiguous())

    @staticmethod
    def magic_mix_range(num_inference_steps: int, kmin: float, kmax: float) -> T.Tuple[int, int]:
        """(t_max, t_min) of Magic Mix: n - int(kmax * n) and n - int(kmin * n), indices into scheduler.timesteps.  The
        loop starts at timesteps[t_max]; steps t_max + 1 .. t_min - 1 are the layout phase."""
        n = num_inference_steps
        if int(kmax * n) < 1:
            raise ValueError(f"kmax * num_inference_steps must be at least 1 (kmax {kmax}, {n} steps): no step would run")
        if kmax > 1.0:
            raise ValueError(f"kmax must be at most 1, got {kmax}")
        return n - int(kmax * n), n - int(kmin * n)

    @staticmethod
    def _check_magic_mix_scheduler(scheduler: str) -> None:
        if scheduler == "EulerAncestralDiscreteScheduler":
            raise ValueError("Magic Mix does not run EulerAncestralDiscreteScheduler: its layout blend noises in "
                             "alpha-bar space, which a sigma-space scheduler does not use")

    @torch.no_grad()
    def magic_mix(self, prompt: str, images: T.Union[None, torch.Tensor, T.Sequence[Image.Image]], *, kmin: float = 0.3,
                  kmax: float = 0.5, mix_factor: float = 0.5, num_inference_steps: int = 25, guidance_scale: float = 7.0,
                  seed: int = 42, scheduler: str = "DPMSolverMultistepScheduler", output_type: T.Optional[str] = "pil",
                  text_embeddings: T.Optional[torch.Tensor] = None, uncond_embeddings: T.Optional[torch.Tensor] = None,
                  noise: T.Optional[torch.Tensor] = None,
                  moments: T.Optional[T.Tuple[torch.Tensor, torch.Tensor]] = None) -> T.Dict[str, T.Any]:
        """Magic Mix (Liew et al. 2022): restyle images with a prompt while keeping their layout, as the reference app's
        "Use Magic Mix" switch runs it (streamlit/util.py:302-350, diffusers' community `magic_mix` pipeline), for a
        batch of images in one CFG loop.  The algorithm is restated from memory, not pinned against diffusers
        (unpinned).

        With n = num_inference_steps, T = scheduler.timesteps (n entries for DPM-Solver++, n + 1 for PNDM), t_max =
        n - int(kmax * n) and t_min = n - int(kmin * n) (`magic_mix_range`; int(kmax * n) < 1 raises ValueError):
        enc = 0.18215 * posterior sample, x = add_noise(enc, noise, T[t_max]), then for every i >= t_max one CFG UNet
        evaluation of u and one scheduler step of x, where u = mix_factor * x + (1 - mix_factor) * add_noise(enc, noise,
        T[i]) in the layout phase t_max < i < t_min and u = x otherwise (`tc_ops.magic_mix`).  kmin >= kmax leaves no
        layout phase: img2img started at T[t_max].

        `noise` is torch.randn((1, 4, h, w)) in fp32 from a CPU generator seeded with `seed`, the same for every image
        (the community pipeline's torch.manual_seed(seed)), and stays fp32.  Image i draws its posterior noise from its
        own CUDA generator seeded with `seed`, as in `img2img` (the community pipeline uses the global CUDA RNG).  The
        unconditional context is embed_text(""): Magic Mix has no negative prompt.  `images`, `moments`,
        `text_embeddings`, `uncond_embeddings`, `scheduler` and `output_type` work as in `img2img`; an injected `noise`
        is (1 or B, 4, h, w).  Returns dict(images, latents (1/0.18215-scaled), latents_unscaled, n_unet_evals, t_max,
        t_min); n_unet_evals = len(T) - t_max.  DDIM runs like PNDM; Euler ancestral is refused (ValueError) before any
        device work: the layout blend noises in ᾱ space, and how the community pipeline treats a sigma-space scheduler is
        not known."""
        self._check_magic_mix_scheduler(scheduler)
        t_max, t_min = self.magic_mix_range(num_inference_steps, kmin, kmax)
        sched = make_scheduler(scheduler)
        sched.set_timesteps(num_inference_steps)
        dev = self._device
        mean, logvar = self._image_moments(images, moments)
        n = mean.shape[0]
        context = self._context(prompt, None, n, guidance_scale > 1.0, text_embeddings, uncond_embeddings)
        enc = torch.cat([_sample_latents(mean[i:i + 1], logvar[i:i + 1],
                                         torch.Generator(device=self.device).manual_seed(seed)) for i in range(n)])
        enc = enc.to(device=dev, dtype=torch.float16).contiguous()
        if noise is None:
            noise = torch.randn((1,) + tuple(enc.shape[1:]), generator=torch.Generator().manual_seed(seed))
        noise = noise.to(device=dev, dtype=torch.float32)
        if noise.dim() != 4 or noise.shape[0] not in (1, n) or noise.shape[1:] != enc.shape[1:]:
            raise ValueError(f"noise must be (1 or {n}, {', '.join(map(str, enc.shape[1:]))}), got {tuple(noise.shape)}")
        noise = noise.expand_as(enc).contiguous()
        timesteps = sched.timesteps[t_max:]
        a = float(sched.alphas_cumprod[int(timesteps[0])])
        latents = ops.magic_mix(enc, enc, noise, a ** 0.5, (1.0 - a) ** 0.5, 0.0)           # mix 0: add_noise at T[t_max]
        latents, n_evals = self._denoise(sched, timesteps, latents, context, guidance_scale,
                                         layout=(mix_factor, enc, noise, t_min - t_max))
        out = self._finish(latents, n_evals, output_type)
        out["t_max"], out["t_min"] = t_max, t_min
        return out

    @torch.no_grad()
    def text_to_audio(self, prompt: str, *, params=None, negative_prompt: T.Optional[str] = None, seed: int = 42,
                      num_clips: int = 1, num_inference_steps: int = 30, guidance_scale: float = 7.0, width: int = 512,
                      height: T.Optional[int] = None, scheduler: str = "DPMSolverMultistepScheduler",
                      text_embeddings: T.Optional[torch.Tensor] = None, uncond_embeddings: T.Optional[torch.Tensor] = None,
                      latents: T.Optional[torch.Tensor] = None, converter=None,
                      init_angles: T.Optional[torch.Tensor] = None,
                      step_noise: T.Optional[torch.Tensor] = None, loop: bool = False) -> T.Dict[str, torch.Tensor]:
        """Text to audio on the device: `txt2img` with height = params.num_frequencies, then VAE decode -> uint8 image ->
        mel amplitudes (`audio_from_spectrogram_image` semantics: R plane for mono, G and B for stereo, max_value 30e6)
        -> inverse mel + Griffin-Lim.  `params` defaults to mono 0-10 kHz; `scheduler`, `latents` and `step_noise` are
        txt2img's.  Returns device tensors: images (B, H, W, 3)
        uint8, waveform (B, channels, hop * (W - 1)) fp32 before peak normalisation, latents, latents_unscaled,
        n_unet_evals.

        `loop` renders a seamless loop: txt2img's `loop` (circular width padding in the UNet and the VAE decoder), then
        the periodic Griffin-Lim (`waveform_from_mel_amplitudes(periodic=True)`), whose waveform of exactly hop * W
        samples per channel plays on repeat without a seam."""
        params = DEFAULT_PARAMS if params is None else params
        if height is not None and height != params.num_frequencies:
            raise ValueError(f"height {height} differs from params.num_frequencies {params.num_frequencies}")
        converter = self._converter(params, converter)
        out = self.txt2img(prompt, negative_prompt=negative_prompt, seed=seed, num_clips=num_clips,
                           num_inference_steps=num_inference_steps, guidance_scale=guidance_scale, width=width,
                           height=params.num_frequencies, scheduler=scheduler, output_type="latent",
                           text_embeddings=text_embeddings, uncond_embeddings=uncond_embeddings, latents=latents,
                           step_noise=step_noise, **(dict(loop=True) if loop else {}))
        if loop:
            u8 = self._decode_u8(out["latents"], True)
            wave = self._u8_to_waveform(u8, converter, params.stereo, init_angles, periodic=True)
        else:
            u8 = self._decode_u8(out["latents"])
            wave = self._u8_to_waveform(u8, converter, params.stereo, init_angles)
        return dict(images=u8, waveform=wave, latents=out["latents"], latents_unscaled=out["latents_unscaled"],
                    n_unet_evals=out["n_unet_evals"])

    # ------------------------------------------------------------------------------ long tracks
    @staticmethod
    def track_loops(num_tracks: int, n_windows: int, max_batch: int) -> T.List[T.List[int]]:
        """The tracks of each CFG loop of `txt2img_track`, in order: as many whole tracks as fit in `max_batch` windows,
        at least one per loop (a track is never split)."""
        if num_tracks < 1:
            raise ValueError("num_tracks must be at least 1")
        if max_batch < 1:
            raise ValueError("max_batch must be at least 1")
        per = max(1, max_batch // n_windows)
        return [list(range(lo, min(num_tracks, lo + per))) for lo in range(0, num_tracks, per)]

    @torch.no_grad()
    def txt2img_track(self, prompt: T.Union[str, T.Sequence[str]], *, width: int, height: int = 512,
                      window_width: int = 512, stride: int = 256, negative_prompt: T.Optional[str] = None, seed: int = 42,
                      num_tracks: int = 1, num_inference_steps: int = 30, guidance_scale: float = 7.0,
                      scheduler: str = "DPMSolverMultistepScheduler", max_batch: int = 32,
                      output_type: T.Optional[str] = "pil", text_embeddings: T.Optional[torch.Tensor] = None,
                      uncond_embeddings: T.Optional[torch.Tensor] = None, latents: T.Optional[torch.Tensor] = None,
                      step_noise: T.Optional[torch.Tensor] = None) -> T.Dict[str, T.Any]:
        """`txt2img` of a canvas wider than the model, MultiDiffusion style (Bar-Tal et al. 2023): the canvas of `width`
        pixels is denoised as n = (width - window_width) / stride + 1 overlapping windows of `window_width` pixels.  Every
        step gathers the windows, runs the UNet on them at its trained size, merges the [uncond | text] eps of the
        windows onto the canvas with the crossfade weights of `window_ops.merge_weights`, and steps the canvas with the
        scheduler's own fused guidance + update (`_denoise` with `windows`).

        `prompt` is one string, or one per window (window k's text context); the prompts and the negative prompt
        (default "") are embedded without weighting.  Track i starts from txt2img's draw at `width` for seed + i, and
        Euler ancestral draws txt2img's per-step noise.  Tracks share loops in order (`track_loops`), so the UNet batch
        is twice the windows of a loop.  `text_embeddings` (1 or n rows) / `uncond_embeddings` / `latents` (num_tracks,
        4, height/8, width/8) / `step_noise` (steps, num_tracks, 4, height/8, width/8) replace the text encoder and the
        generator draws.  With one window the call is `txt2img` at that width.

        Raises ValueError before any device work unless width, window_width, stride and height are positive multiples
        of 64 with 0 < stride <= window_width and width = window_width + (n - 1) stride, for a prompt list that is not one
        per window, num_tracks or max_batch below 1, or an unknown scheduler.  Returns txt2img's dict (n_unet_evals:
        the UNet evaluations of all loops) plus windows (the window offsets in pixels) and loops (the tracks of each
        loop)."""
        n = window_ops.window_count(width, window_width, stride)
        if height <= 0 or height % 64:
            raise ValueError(f"height must be a positive multiple of 64, got {height}")
        prompts = [prompt] * n if isinstance(prompt, str) else list(prompt)
        if len(prompts) != n:
            raise ValueError(f"{len(prompts)} prompts for {n} windows: give one prompt, or one per window")
        loops = self.track_loops(num_tracks, n, max_batch)
        make_scheduler(scheduler)
        dev = self._device
        win = window_ops.Windows.make(window_width // 8, stride // 8, n, dev)
        if text_embeddings is None:
            embedded = {p: self.embed_text(p) for p in dict.fromkeys(prompts)}
            text_embeddings = torch.cat([embedded[p] for p in prompts])
        texts = text_embeddings.to(device=dev, dtype=torch.float16)
        texts = texts.expand(n, -1, -1) if texts.shape[0] == 1 else texts
        if texts.shape[0] != n:
            raise ValueError(f"text_embeddings hold {texts.shape[0]} rows for {n} windows")
        shape = (1, 4, height // 8, width // 8)
        gens = [torch.Generator(device=self.device).manual_seed(seed + i) for i in range(num_tracks)]
        if latents is None:
            latents = torch.cat([torch.randn(shape, generator=g, device=self.device, dtype=torch.float16) for g in gens])
        latents = latents.to(device=dev, dtype=torch.float16).contiguous()
        if tuple(latents.shape) != (num_tracks,) + shape[1:]:
            raise ValueError(f"latents must be {(num_tracks,) + shape[1:]}, got {tuple(latents.shape)}")
        outs, n_evals = [], 0
        for idx in loops:
            sched = make_scheduler(scheduler)
            sched.set_timesteps(num_inference_steps)
            lat = latents[idx[0]:idx[-1] + 1]
            noise = None if step_noise is None else step_noise[:, idx[0]:idx[-1] + 1]
            self._step_noise(sched, len(sched.timesteps), lat, noise, [gens[i] for i in idx])
            if sched.init_noise_sigma != 1.0:
                lat = (lat * sched.init_noise_sigma).contiguous()
            context = self._context(None, negative_prompt, len(idx) * n, guidance_scale > 1.0, texts.repeat(len(idx), 1, 1),
                                    uncond_embeddings)
            lat, evals = self._denoise(sched, sched.timesteps, lat, context, guidance_scale, windows=win)
            outs.append(lat)
            n_evals += evals
        out = self._finish(torch.cat(outs), n_evals, output_type)
        out["windows"] = window_ops.window_offsets(n, stride)
        out["loops"] = loops
        return out

    @staticmethod
    def track_geometry(duration_s: float, window_width: int, stride: int, hop_length: int,
                       sample_rate: int) -> T.Tuple[int, int, int]:
        """(frames, canvas width, windows) of a `duration_s` track: F = ceil(duration_s sr / hop) + 1 frames on the
        narrowest canvas of whole strides that holds them (`window_ops.canvas_width`).  ValueError unless 0 < duration_s
        <= 120 and window_width, stride are positive multiples of 64 with stride <= window_width."""
        if not 0 < duration_s <= 120:
            raise ValueError(f"duration_s must be in (0, 120] seconds, got {duration_s}")
        window_ops.window_count(window_width, window_width, stride)
        frames = math.ceil(duration_s * sample_rate / hop_length) + 1
        width = window_ops.canvas_width(frames, window_width, stride)
        return frames, width, window_ops.window_count(width, window_width, stride)

    @staticmethod
    def track_prompts(prompt: T.Union[str, T.Sequence[T.Tuple[float, str]]], n_windows: int, window_width: int,
                      stride: int, hop_length: int, sample_rate: int) -> T.List[str]:
        """The prompt of each window: `prompt` itself, or from a list of (start_s, prompt) spans, the span in force at
        the window's centre time (k stride + window_width / 2 frames).  ValueError for an empty list or spans whose first
        start is not 0 or whose starts do not strictly increase."""
        if isinstance(prompt, str):
            return [prompt] * n_windows
        spans = [(float(s), p) for s, p in prompt]
        if not spans:
            raise ValueError("no prompt spans: give a prompt or a list of (start_s, prompt)")
        if spans[0][0] != 0.0:
            raise ValueError(f"the first prompt span must start at 0 s, got {spans[0][0]}")
        for (a, _), (b, _) in zip(spans, spans[1:]):
            if not b > a:
                raise ValueError(f"prompt span starts must strictly increase, got {a} then {b}")
        out = []
        for k in range(n_windows):
            centre = (k * stride + window_width / 2) * hop_length / sample_rate
            out.append([p for s, p in spans if s <= centre][-1])
        return out

    @torch.no_grad()
    def text_to_track(self, prompt: T.Union[str, T.Sequence[T.Tuple[float, str]]], *, duration_s: float = 30.0,
                      params=None, window_width: int = 512, stride: int = 256, negative_prompt: T.Optional[str] = None,
                      seed: int = 42, num_tracks: int = 1, num_inference_steps: int = 30, guidance_scale: float = 7.0,
                      scheduler: str = "DPMSolverMultistepScheduler", max_batch: int = 32,
                      text_embeddings: T.Optional[torch.Tensor] = None, uncond_embeddings: T.Optional[torch.Tensor] = None,
                      latents: T.Optional[torch.Tensor] = None, step_noise: T.Optional[torch.Tensor] = None,
                      converter=None, init_angles: T.Optional[torch.Tensor] = None) -> T.Dict[str, T.Any]:
        """A track of `duration_s` seconds from text: `txt2img_track` at height params.num_frequencies on the canvas of
        `track_geometry`, then per track on the device: VAE decode -> uint8 image -> mel (`rf_image_to_mel`) -> inverse
        mel + Griffin-Lim, trimmed to round(duration_s sr) samples.  `params` defaults to mono 0-10 kHz.

        `prompt` is a string or a list of (start_s, prompt) spans (`track_prompts`): each window takes the prompt in force
        at its centre, so the overlaps crossfade from one prompt to the next.  `init_angles` (num_tracks, channels,
        n_fft/2 + 1, canvas width) fixes Griffin-Lim's initial phases; the other options are `txt2img_track`'s.

        Raises ValueError before any device work for a duration outside (0, 120] s, bad window geometry, malformed
        prompt spans, an unknown scheduler, num_tracks or max_batch below 1.  Returns device tensors images
        (num_tracks, H, canvas width, 3) uint8, waveform (num_tracks, channels, round(duration_s sr)) fp32 before peak
        normalisation, latents, latents_unscaled, and windows (per window: offset in pixels and prompt), n_unet_evals,
        loops."""
        params = DEFAULT_PARAMS if params is None else params
        hop, sr = params.hop_length, params.sample_rate
        _, width, n = self.track_geometry(duration_s, window_width, stride, hop, sr)
        prompts = self.track_prompts(prompt, n, window_width, stride, hop, sr)
        self.track_loops(num_tracks, n, max_batch)
        make_scheduler(scheduler)
        converter = self._converter(params, converter)
        out = self.txt2img_track(prompts, width=width, height=params.num_frequencies, window_width=window_width,
                                 stride=stride, negative_prompt=negative_prompt, seed=seed, num_tracks=num_tracks,
                                 num_inference_steps=num_inference_steps, guidance_scale=guidance_scale,
                                 scheduler=scheduler, max_batch=max_batch, output_type="latent",
                                 text_embeddings=text_embeddings, uncond_embeddings=uncond_embeddings, latents=latents,
                                 step_noise=step_noise)
        samples = round(duration_s * sr)
        u8s, waves = [], []
        for i in range(num_tracks):
            u8 = self._decode_u8(out["latents"][i:i + 1])
            angles = None if init_angles is None else init_angles[i:i + 1]
            waves.append(self._u8_to_waveform(u8, converter, params.stereo, angles)[..., :samples])
            u8s.append(u8)
        return dict(images=torch.cat(u8s), waveform=torch.cat(waves), latents=out["latents"],
                    latents_unscaled=out["latents_unscaled"],
                    windows=[dict(offset=o, prompt=p) for o, p in zip(out["windows"], prompts)],
                    n_unet_evals=out["n_unet_evals"], loops=out["loops"])

    @torch.no_grad()
    def text_to_audio_batch(self, batch: dict, *, num_seeds: int = 1, max_batch: int = 32, converter=None,
                            apply_filters: bool = True) -> T.Dict[str, T.Any]:
        """The app's Text to Audio Batch task (streamlit/tasks/text_to_audio_batch.py) on a loaded batch JSON object
        (format: `riffusion.text_to_audio_batch`).  For every (entry, seed, param set), in that order, the clip is
        `txt2img` of the entry's prompt / negative prompt at that seed with the set's steps, guidance, width and
        scheduler, at height 512, turned into mono 0-10 kHz audio.  The param sets' `checkpoint` is not loaded: every
        clip runs on this pipeline.

        Clips are grouped into loops by `text_to_audio_batch.plan_batch` (same scheduler, steps, width and side of
        guidance 1; at most `max_batch` rows), and each loop is one CFG loop whose rows keep their own guidance
        (`DPMSolverRowsB200`, `PNDMRowsB200` for PNDM and DDIM, `EulerAncestralRowsB200`).  Row r starts from
        `torch.randn((1, 4, 64, W/8))` drawn from a CUDA generator seeded with its seed (then, for Euler ancestral, one
        draw per step from the same generator), with context [embed_text(negative or "") | embed_text(prompt)], exactly
        txt2img's draws.  After each loop, on the device: VAE decode -> uint8 image -> mel -> waveform; on the host:
        peak-normalised int16 and, with `apply_filters`, `apply_filters(compression=False)`.

        Raises ValueError before any device work for a malformed batch, num_seeds or max_batch below 1.  Returns
        dict(clips, loops): per clip (in the app's order) param_index, param_name, entry_index, seed, prompt,
        negative_prompt, latents_unscaled ((4, 64, W/8) fp16, the loop's output), image ((512, W, 3) uint8), waveform
        ((1, L) fp32 before normalisation), all device tensors, and segment (AudioSegment); per loop rows (clip
        indices), scheduler, num_inference_steps, width, n_unet_evals."""
        from riffusion.scheduler_b200 import SCHEDULERS, DPMSolverRowsB200, EulerAncestralRowsB200, PNDMRowsB200
        from riffusion.text_to_audio_batch import parse_batch, plan_batch
        from riffusion.util import audio_util

        param_sets, entries = parse_batch(batch)
        clips, loops = plan_batch(param_sets, entries, num_seeds, max_batch)
        params = DEFAULT_PARAMS
        converter = self._converter(params, converter)
        out_clips: T.List[T.Optional[dict]] = [None] * len(clips)
        out_loops = []
        for loop in loops:
            rows = [clips[k] for k in loop.rows]
            guidances = [param_sets[c.param_index].guidance for c in rows]
            texts = torch.cat([self.embed_text(entries[c.entry_index].prompt) for c in rows])
            unconds = torch.cat([self.embed_text(entries[c.entry_index].negative_prompt or "") for c in rows])
            context = self._context(None, None, len(rows), loop.cfg, texts, unconds)
            shape = (1, 4, params.num_frequencies // 8, loop.width // 8)
            gens = [torch.Generator(device=self.device).manual_seed(c.seed) for c in rows]
            latents = torch.cat([torch.randn(shape, generator=g, device=self.device, dtype=torch.float16)
                                 for g in gens]).contiguous()
            if loop.scheduler in ("PNDMScheduler", "DDIMScheduler"):
                sched = PNDMRowsB200(loop.num_inference_steps, [0] * len(rows), guidances, device=self._device,
                                     scheduler=SCHEDULERS[loop.scheduler])
            elif loop.scheduler == "EulerAncestralDiscreteScheduler":
                sched = EulerAncestralRowsB200(loop.num_inference_steps, guidances, device=self._device)
                self._step_noise(sched, len(sched.timesteps), latents, None, gens)
                latents = (latents * sched.init_noise_sigma).contiguous()
            else:
                sched = DPMSolverRowsB200(loop.num_inference_steps, guidances, device=self._device)
            latents, n_evals = self._denoise(sched, sched.timesteps, latents, context, guidances[0])
            u8 = self._decode_u8((1.0 / VAE_SCALE) * latents)
            wave = self._u8_to_waveform(u8, converter, params.stereo, None)
            for j, (k, c) in enumerate(zip(loop.rows, rows)):
                seg = audio_util.audio_from_waveform(samples=wave[j].cpu().numpy(), sample_rate=params.sample_rate,
                                                     normalize=True)
                entry = entries[c.entry_index]
                out_clips[k] = dict(param_index=c.param_index, param_name=param_sets[c.param_index].name,
                                    entry_index=c.entry_index, seed=c.seed, prompt=entry.prompt,
                                    negative_prompt=entry.negative_prompt, latents_unscaled=latents[j], image=u8[j],
                                    waveform=wave[j],
                                    segment=audio_util.apply_filters(seg, compression=False) if apply_filters else seg)
            out_loops.append(dict(rows=list(loop.rows), scheduler=loop.scheduler,
                                  num_inference_steps=loop.num_inference_steps, width=loop.width, n_unet_evals=n_evals))
        return dict(clips=out_clips, loops=out_loops)

    def _converter(self, params, converter):
        """`converter`, which must have been built for `params`, or a new SpectrogramConverter for them on this
        pipeline's device."""
        from riffusion.spectrogram_converter import SpectrogramConverter

        if converter is None:
            converter = SpectrogramConverter(params, device=self.device)
        if converter.p != params:
            raise ValueError("converter was built for other SpectrogramParams")
        return converter

    @staticmethod
    def _u8_to_waveform(u8: torch.Tensor, converter, stereo: bool, init_angles: T.Optional[torch.Tensor],
                        periodic: bool = False) -> torch.Tensor:
        """uint8 images (B, H, W, 3) -> mel amplitudes (B, channels, H, W) -> waveform (B, channels, L); `periodic`: the
        loop Griffin-Lim, L = hop * W."""
        from riffusion import _native

        B, H, W, _ = _native.operand(u8, "u8", torch.uint8, shape=(_native.ANY, _native.ANY, _native.ANY, 3)).shape
        mel = torch.empty((B, 2 if stereo else 1, H, W), dtype=torch.float32, device=u8.device)
        p = converter.p
        for i in range(B):
            _native.call("rf_image_to_mel", u8.device, u8[i].data_ptr(), H, W, int(stereo), float(p.power_for_image),
                         30e6, mel[i].data_ptr())
        if periodic:
            return converter.waveform_from_mel_amplitudes(mel, init_angles, periodic=True)
        return converter.waveform_from_mel_amplitudes(mel, init_angles)

    # ------------------------------------------------------------------------------ audio -> audio
    @torch.no_grad()
    def audio_to_audio(self, track, prompt: str, *, params=None, start_time_s: float = 0.0, duration_s: float = 20.0,
                       clip_duration_s: float = 5.0, overlap_duration_s: float = 0.2,
                       negative_prompt: T.Optional[str] = None, seed: int = 42, denoising: float = 0.55,
                       num_inference_steps: int = 25, guidance_scale: float = 7.0,
                       scheduler: str = "DPMSolverMultistepScheduler", prompt_b: T.Optional[str] = None,
                       seed_b: T.Optional[int] = None, denoising_b: T.Optional[float] = None, max_batch: int = 32,
                       init_angles: T.Optional[torch.Tensor] = None, apply_filters: bool = True,
                       text_embeddings: T.Optional[torch.Tensor] = None,
                       uncond_embeddings: T.Optional[torch.Tensor] = None, converter=None, magic_mix: bool = False,
                       kmin: float = 0.3, kmax: float = 0.5, mix_factor: float = 0.5) -> T.Dict[str, T.Any]:
        """Riff a whole track: the reference app's Audio to Audio task (streamlit/tasks/audio_to_audio.py:86-330).

        The track (an AudioSegment at params.sample_rate) is cut into overlapping clips (`audio_to_audio.clip_start_times`,
        `slice_audio_into_clips`).  On the device, per batch of at most `max_batch` clips: waveform -> mel -> uint8 image
        (per-clip max, `spectrogram_image_from_audio`), bicubic resize to a 32-pixel stride -> VAE encode -> img2img ->
        VAE decode -> uint8 -> bicubic resize back -> mel -> waveform.  On the host: peak-normalised int16,
        `apply_filters` and `stitch_segments` with an `overlap_duration_s` crossfade.

        `params` defaults to mono 0-10 kHz.  Without `prompt_b` every clip runs `img2img` (prompt, negative prompt,
        `denoising` as strength, `seed` for every clip, `scheduler`).  With `prompt_b` it is the interpolation mode: clip i
        of n is `riffuse_batch` of InferenceInput(alpha = linspace(0, 1, n)[i], start = (prompt, seed, denoising),
        end = (prompt_b, seed_b, denoising_b)) - PNDM, weighted prompts, no negative prompt.  `init_angles` (clips,
        channels, n_fft/2 + 1, frames) fixes Griffin-Lim's initial phases; `text_embeddings` / `uncond_embeddings`
        replace the text encoder of the img2img and Magic Mix modes.  With `magic_mix` every batch runs `magic_mix`
        (prompt, `kmin`, `kmax`, `mix_factor`, `seed`, `scheduler`; `denoising` is not used) in place of `img2img`; it
        cannot be combined with `prompt_b` or a negative prompt (ValueError), as in the app.

        Returns dict(segment (the stitched AudioSegment), source_images and images ((clips, H, W, 3) uint8 device tensors
        before and after denoising), denoised_images (the decoded images at the 32-stride size), clip_start_times (s), waveform ((clips, channels, L) fp32, before normalisation),
        n_unet_evals (per batch))."""
        from riffusion import audio_to_audio as a2a
        from riffusion.datatypes import PromptInput
        from riffusion.spectrogram_image_converter import _conform_channels
        from riffusion.util import audio_util, image_util

        params = DEFAULT_PARAMS if params is None else params
        if max_batch < 1:
            raise ValueError("max_batch must be at least 1")
        if magic_mix and prompt_b is not None:
            raise ValueError("magic_mix cannot be combined with interpolation (prompt_b)")
        if magic_mix and negative_prompt:
            raise ValueError("magic_mix takes no negative prompt")
        if magic_mix:
            self._check_magic_mix_scheduler(scheduler)
            self.magic_mix_range(num_inference_steps, kmin, kmax)          # its ValueError before any device work
        if track.frame_rate != params.sample_rate:
            track = track.set_frame_rate(params.sample_rate)        # the app resamples (audio_to_audio.py:89-91)
        starts = a2a.clip_start_times(track.duration_seconds, start_time_s, duration_s, clip_duration_s,
                                      overlap_duration_s)
        if len(starts) == 0:
            raise ValueError(f"no {clip_duration_s} s clip fits in {track.duration_seconds:.2f} s of audio from "
                             f"{start_time_s} s (duration {duration_s} s): the track is shorter than one clip")
        frames = a2a.clip_frames(clip_duration_s, params.sample_rate, params.hop_length)
        width, height = a2a.stride_32_size(frames, params.num_frequencies)
        a2a.check_denoising_size(width, height, clip_duration_s)
        converter = self._converter(params, converter)

        clips = [_conform_channels(c, params.stereo) for c in a2a.slice_audio_into_clips(track, starts, clip_duration_s)]
        waves = np.stack([np.array([c.get_array_of_samples() for c in clip.split_to_mono()]) for clip in clips])
        waves = torch.from_numpy(waves.astype(np.float32)).to(self._device)           # (clips, channels, samples)
        n = waves.shape[0]
        if prompt_b is not None:
            alphas = np.linspace(0, 1, n)
            a = PromptInput(prompt=prompt, seed=seed, denoising=denoising, guidance=guidance_scale)
            b = PromptInput(prompt=prompt_b, seed=seed if seed_b is None else seed_b,
                            denoising=denoising if denoising_b is None else denoising_b, guidance=guidance_scale)
            requests = [InferenceInput(start=a, end=b, alpha=float(al), num_inference_steps=num_inference_steps)
                        for al in alphas]
        sources, denoised, riffed, out_waves, n_evals = [], [], [], [], []
        for lo in range(0, n, max_batch):
            hi = min(n, lo + max_batch)
            mel = converter.mel_amplitudes_from_waveform(waves[lo:hi])                 # (b, channels, H, frames)
            src = torch.stack([image_util.image_from_spectrogram_device(m, power=params.power_for_image)[0] for m in mel])
            Hs, Ws = src.shape[1], src.shape[2]
            _, vae_in = ops.resize_bicubic_u8(src, width, height, want_f16=True)
            moments = self.vae.encode_moments(vae_in)
            if prompt_b is None:
                if magic_mix:
                    out = self.magic_mix(prompt, None, kmin=kmin, kmax=kmax, mix_factor=mix_factor,
                                         num_inference_steps=num_inference_steps, guidance_scale=guidance_scale,
                                         seed=seed, scheduler=scheduler, output_type="latent",
                                         text_embeddings=text_embeddings, uncond_embeddings=uncond_embeddings,
                                         moments=moments)
                else:
                    out = self.img2img(prompt, None, strength=denoising, num_inference_steps=num_inference_steps,
                                       guidance_scale=guidance_scale, negative_prompt=negative_prompt, seed=seed,
                                       scheduler=scheduler, output_type="latent", text_embeddings=text_embeddings,
                                       uncond_embeddings=uncond_embeddings, moments=moments)
                latents = out["latents"]
                n_evals.append(out["n_unet_evals"])
            else:
                latents = torch.cat(self.riffuse_batch(requests[lo:hi], None, moments=moments, output_type="latent"))
            u8 = self._decode_u8(latents)
            back, _ = ops.resize_bicubic_u8(u8, Ws, Hs)
            angles = None if init_angles is None else init_angles[lo:hi]
            out_waves.append(self._u8_to_waveform(back, converter, params.stereo, angles))
            sources.append(src)
            denoised.append(u8)
            riffed.append(back)
        waveform = torch.cat(out_waves)
        segments = []
        for w in waveform.cpu().numpy():
            seg = audio_util.audio_from_waveform(samples=w, sample_rate=params.sample_rate, normalize=True)
            segments.append(audio_util.apply_filters(seg, compression=False) if apply_filters else seg)
        return dict(segment=audio_util.stitch_segments(segments, crossfade_s=overlap_duration_s),
                    source_images=torch.cat(sources), denoised_images=torch.cat(denoised), images=torch.cat(riffed),
                    clip_start_times=starts,
                    waveform=waveform, n_unet_evals=n_evals)

    # ------------------------------------------------------------------------------ batched request -> audio
    @torch.no_grad()
    def generate_clips(self, text_embeddings: torch.Tensor, uncond_embeddings: torch.Tensor, init_latents: torch.Tensor,
                       noise: torch.Tensor, strength: float, num_inference_steps: int, guidance_scale: float,
                       converter, init_angles: T.Optional[torch.Tensor] = None) -> T.Dict[str, torch.Tensor]:
        """B independent requests end to end on the device (SURVEY 8(f)-1/2): denoise -> VAE decode -> uint8 image ->
        mel amplitudes (image_util.spectrogram_from_image semantics, mono = R plane) -> inverse mel + Griffin-Lim.
        This is what `server.compute_request` does per request (riffuse, then audio_from_spectrogram_image,
        server.py:145-164) without leaving the GPU in between.  Returns device tensors:
        images (B,512,512,3) uint8, waveform (B, L) fp32, latents."""
        out = self.interpolate_img2img(
            text_embeddings=text_embeddings, init_latents=init_latents, generator_a=None, generator_b=None,
            interpolate_alpha=0.0, strength_a=strength, strength_b=strength, num_inference_steps=num_inference_steps,
            guidance_scale=guidance_scale, uncond_embeddings=uncond_embeddings, noise=noise, output_type="latent")
        u8 = self._decode_u8(out["latents"])
        wave = self._u8_to_waveform(u8, converter, False, init_angles)
        return dict(images=u8, waveform=wave[:, 0], latents=out["latents"], latents_unscaled=out["latents_unscaled"],
                    n_unet_evals=out["n_unet_evals"])

    @staticmethod
    def numpy_to_pil(images: np.ndarray) -> T.List[Image.Image]:
        """diffusers DiffusionPipeline.numpy_to_pil: (x * 255).round().astype(uint8)"""
        if images.ndim == 3:
            images = images[None, ...]
        images = (images * 255).round().astype("uint8")
        return [Image.fromarray(im) for im in images]

    def progress_bar(self, iterable):
        return iterable


def _load_weights(folder: Path) -> T.Dict[str, torch.Tensor]:
    for name in ("diffusion_pytorch_model.safetensors", "model.safetensors"):
        f = folder / name
        if f.exists():
            from safetensors.torch import load_file

            return load_file(str(f))
    for name in ("diffusion_pytorch_model.bin", "pytorch_model.bin"):
        f = folder / name
        if f.exists():
            return torch.load(str(f), map_location="cpu", weights_only=True)
    raise FileNotFoundError(f"no diffusers weight file under {folder}")


def _sample_latents(mean: torch.Tensor, logvar: torch.Tensor, generator: torch.Generator) -> torch.Tensor:
    """0.18215 * a sample of the VAE posterior with these moments, its fp32 noise drawn from `generator` (:259-264)."""
    return VAE_SCALE * _Posterior(mean, logvar).sample(generator=generator)


def preprocess_image(image: Image.Image) -> torch.Tensor:
    """PIL RGB -> (1, 3, H, W) float in [-1, 1], size rounded down to multiples of 32 with LANCZOS
    (riffusion_pipeline.py:439-452)."""
    w, h = image.size
    w, h = (x - x % 32 for x in (w, h))
    image = image.resize((w, h), resample=Image.LANCZOS)
    arr = np.array(image).astype(np.float32) / 255.0
    arr = arr[None].transpose(0, 3, 1, 2)
    return 2.0 * torch.from_numpy(arr) - 1.0


def preprocess_mask(mask: Image.Image, scale_factor: int = 8) -> torch.Tensor:
    """PIL mask -> (1, 4, h/8, w/8) with white = repaint (riffusion_pipeline.py:455-477)."""
    mask = mask.convert("L")
    w, h = mask.size
    w, h = (x - x % 32 for x in (w, h))
    mask = mask.resize((w // scale_factor, h // scale_factor), resample=Image.NEAREST)
    arr = np.array(mask).astype(np.float32) / 255.0
    arr = np.tile(arr, (4, 1, 1))[None]          # the reference's transpose(0,1,2,3) is a no-op
    return torch.from_numpy(1 - arr)
