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
import inspect
import typing as T
from pathlib import Path

import numpy as np
import torch
from PIL import Image

from riffusion import tc_ops as ops
from riffusion.datatypes import InferenceInput
from riffusion.scheduler_b200 import PNDMSchedulerB200, make_scheduler
from riffusion.unet_b200 import UNetB200
from riffusion.util import torch_util
from riffusion.vae_b200 import VaeB200

VAE_SCALE = 0.18215


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
    def riffuse_batch(self, inputs: T.Sequence[InferenceInput], init_images: T.Union[Image.Image, T.Sequence[Image.Image]],
                      mask_image: T.Optional[Image.Image] = None, use_reweighting: bool = True) -> T.List[Image.Image]:
        """`riffuse` for a list of requests in one batched denoising loop (SURVEY 8(f)-2) — what
        streamlit/tasks/interpolation.py:146-164 does one request at a time.  Every request draws exactly what `riffuse`
        draws for it (posterior noise and noise_a from generator(start.seed), noise_b from generator(end.seed), per-request
        alpha for the slerp and the prompt interpolation), so result i equals `riffuse(inputs[i], ...)` up to the batch-size
        dependent accumulation order of the kernels.  Requests are grouped by (strength, guidance, steps): the PNDM state
        and the guidance scalar are shared inside a group."""
        images = [init_images] * len(inputs) if isinstance(init_images, Image.Image) else list(init_images)
        assert len(images) == len(inputs)
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
            texts, lats, nas, nbs, alphas = [], [], [], [], []
            for i in idx:
                inp = inputs[i]
                e0, e1 = embed(inp.start.prompt), embed(inp.end.prompt)
                texts.append(e0 + inp.alpha * (e1 - e0))
                lats.append(self.encode_image(images[i], torch.Generator(device=self.device).manual_seed(inp.start.seed)))
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
            out = self.interpolate_img2img(
                text_embeddings=torch.cat(texts), init_latents=torch.cat(lats), mask=mask, generator_a=None, generator_b=None,
                interpolate_alpha=0.0, strength_a=strength, strength_b=strength, num_inference_steps=steps,
                guidance_scale=guidance, noise=noise)
            for j, i in enumerate(idx):
                results[i] = out["images"][j]
        return results  # type: ignore[return-value]

    def encode_image(self, init_image: Image.Image, generator: torch.Generator) -> torch.Tensor:
        """preprocess + VAE posterior sample * 0.18215 (:252-264).  The (mean, logvar) moments only depend on the
        image and are cached; the posterior noise is drawn from `generator` like the reference."""
        key = hash(init_image.tobytes()) ^ hash(init_image.size)
        if key not in self._moment_cache:
            img = preprocess_image(init_image).to(device=self.device, dtype=torch.float16)
            self._moment_cache[key] = self.vae.encode_moments(img)
        mean, logvar = self._moment_cache[key]
        from riffusion.vae_b200 import _Posterior

        return VAE_SCALE * _Posterior(mean, logvar).sample(generator=generator)

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
        the parity tests and by runs without a text encoder."""
        batch_size = text_embeddings.shape[0]
        self.scheduler.set_timesteps(num_inference_steps)
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
            uncond_embeddings = uncond_embeddings.to(device=dev, dtype=torch.float16)
            uncond_embeddings = uncond_embeddings.repeat_interleave(batch_size * num_images_per_prompt // uncond_embeddings.shape[0], dim=0)
            context = torch.cat([uncond_embeddings, text_embeddings]).contiguous()              # :354
        else:
            context = text_embeddings.contiguous()

        latents_dtype = torch.float16
        strength = (1 - interpolate_alpha) * strength_a + interpolate_alpha * strength_b          # :358
        offset = self.scheduler.config.get("steps_offset", 0)
        init_timestep = min(int(num_inference_steps * strength) + offset, num_inference_steps)    # :361-363
        t_noise = int(self.scheduler.timesteps[-init_timestep])                                   # :365
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
        init_latents_orig = init_latents
        latents = self.scheduler.add_noise(init_latents, noise, t_noise)                           # :379

        accepts_eta = "eta" in set(inspect.signature(self.scheduler.step).parameters.keys())       # PNDM ignores eta
        del accepts_eta
        t_start = max(num_inference_steps - init_timestep + offset, 0)                             # :392
        timesteps = self.scheduler.timesteps[t_start:]
        ctx_cache: T.Dict[str, T.Any] = {}
        graphed = self._graphed_unet(latents.shape, context) if do_cfg else None
        n_evals = 0
        for t in timesteps:                                                                        # :398
            t_int = int(t)
            if graphed is not None:
                eps_pair = graphed(latents, t_int)
            else:
                model_in = torch.cat([latents] * 2) if do_cfg else latents                         # :400-403
                eps_pair = self.unet(model_in, t_int, encoder_hidden_states=context, ctx_cache=ctx_cache).sample
            n_evals += 1
            if not do_cfg:
                eps_pair = torch.cat([eps_pair, eps_pair])
            latents = self.scheduler.step_cfg(eps_pair, guidance_scale if do_cfg else 0.0, t_int, latents)   # :411-418
            if mask is not None:                                                                   # :420-425
                m = mask.to(device=dev, dtype=latents_dtype).expand_as(latents).contiguous()
                latents = self.scheduler.add_noise(init_latents_orig, noise, t_int, mask=m, blend_with=latents)

        # :427 — the reference rescales in fp16 (`1.0 / 0.18215 * latents`) and returns THAT tensor under "latents"; the
        # un-scaled loop state and the evaluation count are extra keys of this implementation
        scaled = (1.0 / VAE_SCALE) * latents
        out: T.Dict[str, T.Any] = dict(latents=scaled, nsfw_content_detected=False, latents_unscaled=latents,
                                       n_unet_evals=n_evals)
        if output_type == "latent" or self.vae is None:
            out["images"] = None
            return out
        image = self.vae.decode(scaled).sample                                                       # :428
        if output_type == "pil":
            # :430-434 `(image / 2 + 0.5).clamp(0, 1)` -> numpy_to_pil, in the fp16 arithmetic of the reference's CUDA path
            u8 = ops.vae_image_to_u8(image).cpu().numpy()
            out["images"] = [Image.fromarray(im) for im in u8]
        else:
            out["images"] = (image / 2 + 0.5).clamp(0, 1).cpu().permute(0, 2, 3, 1).numpy()         # float16 array, like the reference
        return out

    def _graphed_unet(self, latent_shape, context: torch.Tensor):
        """The CUDA-graph CFG evaluation for this (latent shape, context shape), or None when graphs are off."""
        if not self.use_cuda_graph:
            return None
        from riffusion.graphed import GraphedUNet

        # one captured graph per (latent shape, context shape); a new request only refreshes the cross-attention
        # K / V^T that the graph reads (capture costs two eager evaluations + instantiation)
        gkey = (tuple(latent_shape), tuple(context.shape))
        graphed = self._graphs.get(gkey)
        if graphed is None:
            graphed = self._graphs[gkey] = GraphedUNet(self.unet, latent_shape, context)
        else:
            graphed.set_context(context)
        return graphed

    # ------------------------------------------------------------------------------ text -> image
    @torch.no_grad()
    def txt2img(self, prompt: str, *, negative_prompt: T.Optional[str] = None, seed: int = 42, num_clips: int = 1,
                num_inference_steps: int = 30, guidance_scale: float = 7.0, width: int = 512, height: int = 512,
                scheduler: str = "DPMSolverMultistepScheduler", output_type: T.Optional[str] = "pil",
                text_embeddings: T.Optional[torch.Tensor] = None, uncond_embeddings: T.Optional[torch.Tensor] = None,
                latents: T.Optional[torch.Tensor] = None) -> T.Dict[str, T.Any]:
        """Text to spectrogram image: Stable Diffusion txt2img, the reference app's text-to-audio generation.

        Clip i starts from `torch.randn((1, 4, height/8, width/8))` drawn from a CUDA generator seeded with `seed + i`
        (one pipeline call per seed in the app); all clips run as one CFG batch.  The prompt and the negative prompt
        (default "") are encoded without prompt weighting.  `scheduler` is "DPMSolverMultistepScheduler" or
        "PNDMScheduler"; a fresh instance is used per call.  `width` and `height` must be multiples of 64 (diffusers
        accepts multiples of 8).  `text_embeddings` / `uncond_embeddings` / `latents` replace the text encoder and the
        generator draws.  Returns dict(images, latents (1/0.18215-scaled), latents_unscaled, n_unet_evals)."""
        if width <= 0 or height <= 0 or width % 64 or height % 64:
            raise ValueError(f"width and height must be positive multiples of 64, got {width}x{height}")
        if num_clips < 1:
            raise ValueError("num_clips must be at least 1")
        sched = make_scheduler(scheduler)
        sched.set_timesteps(num_inference_steps)
        dev = self._device
        do_cfg = guidance_scale > 1.0
        text = self.embed_text(prompt) if text_embeddings is None else text_embeddings
        text = text.to(device=dev, dtype=torch.float16)
        text = text.expand(num_clips, -1, -1) if text.shape[0] == 1 else text
        if text.shape[0] != num_clips:
            raise ValueError(f"text_embeddings hold {text.shape[0]} rows for {num_clips} clips")
        if do_cfg:
            uncond = self.embed_text(negative_prompt or "") if uncond_embeddings is None else uncond_embeddings
            uncond = uncond.to(device=dev, dtype=torch.float16)
            uncond = uncond.expand(num_clips, -1, -1) if uncond.shape[0] == 1 else uncond
            context = torch.cat([uncond, text]).contiguous()
        else:
            context = text.contiguous()
        shape = (1, 4, height // 8, width // 8)
        if latents is None:
            latents = torch.cat([torch.randn(shape, generator=torch.Generator(device=self.device).manual_seed(seed + i),
                                             device=self.device, dtype=torch.float16) for i in range(num_clips)])
        latents = latents.to(device=dev, dtype=torch.float16).contiguous()
        if tuple(latents.shape) != (num_clips,) + shape[1:]:
            raise ValueError(f"latents must be {(num_clips,) + shape[1:]}, got {tuple(latents.shape)}")
        if sched.init_noise_sigma != 1.0:
            latents = (latents * sched.init_noise_sigma).contiguous()

        ctx_cache: T.Dict[str, T.Any] = {}
        graphed = self._graphed_unet(latents.shape, context) if do_cfg else None
        n_evals = 0
        for t in sched.timesteps:
            t_int = int(t)
            if graphed is not None:
                eps_pair = graphed(latents, t_int)
            else:
                model_in = torch.cat([latents] * 2) if do_cfg else latents
                eps_pair = self.unet(model_in, t_int, encoder_hidden_states=context, ctx_cache=ctx_cache).sample
            n_evals += 1
            if not do_cfg:
                eps_pair = torch.cat([eps_pair, eps_pair])
            latents = sched.step_cfg(eps_pair, guidance_scale if do_cfg else 0.0, t_int, latents)

        scaled = (1.0 / VAE_SCALE) * latents
        out: T.Dict[str, T.Any] = dict(latents=scaled, latents_unscaled=latents, n_unet_evals=n_evals)
        if output_type == "latent" or self.vae is None:
            out["images"] = None
            return out
        image = self.vae.decode(scaled).sample
        if output_type == "pil":
            out["images"] = [Image.fromarray(im) for im in ops.vae_image_to_u8(image).cpu().numpy()]
        else:
            out["images"] = (image / 2 + 0.5).clamp(0, 1).cpu().permute(0, 2, 3, 1).numpy()
        return out

    @torch.no_grad()
    def text_to_audio(self, prompt: str, *, params=None, negative_prompt: T.Optional[str] = None, seed: int = 42,
                      num_clips: int = 1, num_inference_steps: int = 30, guidance_scale: float = 7.0, width: int = 512,
                      height: T.Optional[int] = None, scheduler: str = "DPMSolverMultistepScheduler",
                      text_embeddings: T.Optional[torch.Tensor] = None, uncond_embeddings: T.Optional[torch.Tensor] = None,
                      latents: T.Optional[torch.Tensor] = None, converter=None,
                      init_angles: T.Optional[torch.Tensor] = None) -> T.Dict[str, torch.Tensor]:
        """Text to audio on the device: `txt2img` with height = params.num_frequencies, then VAE decode -> uint8 image ->
        mel amplitudes (`audio_from_spectrogram_image` semantics: R plane for mono, G and B for stereo, max_value 30e6)
        -> inverse mel + Griffin-Lim.  `params` defaults to mono 0-10 kHz.  Returns device tensors: images (B, H, W, 3)
        uint8, waveform (B, channels, hop * (W - 1)) fp32 before peak normalisation, latents, latents_unscaled,
        n_unet_evals."""
        from riffusion.spectrogram_converter import SpectrogramConverter
        from riffusion.spectrogram_params import SpectrogramParams

        if params is None:
            params = SpectrogramParams(min_frequency=0, max_frequency=10000, stereo=False)
        if height is not None and height != params.num_frequencies:
            raise ValueError(f"height {height} differs from params.num_frequencies {params.num_frequencies}")
        if converter is None:
            converter = SpectrogramConverter(params, device=self.device)
        if converter.p != params:
            raise ValueError("converter was built for other SpectrogramParams")
        out = self.txt2img(prompt, negative_prompt=negative_prompt, seed=seed, num_clips=num_clips,
                           num_inference_steps=num_inference_steps, guidance_scale=guidance_scale, width=width,
                           height=params.num_frequencies, scheduler=scheduler, output_type="latent",
                           text_embeddings=text_embeddings, uncond_embeddings=uncond_embeddings, latents=latents)
        u8, wave = self._latents_to_audio(out["latents"], converter, params.stereo, init_angles)
        return dict(images=u8, waveform=wave, latents=out["latents"], latents_unscaled=out["latents_unscaled"],
                    n_unet_evals=out["n_unet_evals"])

    def _latents_to_audio(self, scaled_latents: torch.Tensor, converter, stereo: bool,
                          init_angles: T.Optional[torch.Tensor]) -> T.Tuple[torch.Tensor, torch.Tensor]:
        """VAE decode -> uint8 image (B, H, W, 3) -> mel amplitudes (B, channels, H, W) -> waveform (B, channels, L),
        without leaving the device."""
        from riffusion import _native

        image = self.vae.decode(scaled_latents).sample
        u8 = ops.vae_image_to_u8(image)
        B, H, W, _ = u8.shape
        mel = torch.empty((B, 2 if stereo else 1, H, W), dtype=torch.float32, device=u8.device)
        p = converter.p
        for i in range(B):
            _native.call("rf_image_to_mel", u8.device, u8[i].data_ptr(), H, W, int(stereo), float(p.power_for_image),
                         30e6, mel[i].data_ptr())
        return u8, converter.waveform_from_mel_amplitudes(mel, init_angles)

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
        u8, wave = self._latents_to_audio(out["latents"], converter, False, init_angles)
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
