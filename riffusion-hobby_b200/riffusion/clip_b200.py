"""ClipTextB200 — the CLIP text encoder (openai/clip-vit-large-patch14 text tower: 12 layers, width 768, 12 heads, MLP 3072,
quick_gelu, 77 positions, causal attention) on this library's wgmma GEMM / attention kernels (SURVEY §8(f)-3).

Seam: `RiffusionPipeline.embed_text` / `embed_text_weighted` call `self.text_encoder(input_ids)[0]`
(riffusion/riffusion_pipeline.py:177-206, external/prompt_weighting.py:194-234); the reference's object there is
`transformers.CLIPTextModel` (loaded by diffusers' from_pretrained, :92-102).  `ClipTextB200.__call__(input_ids)` returns
`(last_hidden_state,)` like it: (B, 77, 768) fp16 after the final LayerNorm.  Weights: a `CLIPTextModel.state_dict()`
(names `text_model.embeddings.*`, `text_model.encoder.layers.{i}.*`, `text_model.final_layer_norm.*`).

Runs once per distinct prompt (the pipeline lru-caches the result), so this is about being self-contained on the GPU path —
no transformers / cuBLAS call on any path the pipeline takes — not about throughput.  The token / position embedding gather
is a torch indexing op (plumbing); everything else runs in librf_b200.so.
"""
from __future__ import annotations

import typing as T

import torch

from riffusion import tc_ops as ops


class ClipTextB200:
    def __init__(self, state_dict: T.Mapping[str, torch.Tensor], device: str = "cuda", heads: int = 12, eps: float = 1e-5):
        self.device = torch.device(device)
        self.heads, self.eps = heads, eps
        pfx = "text_model." if any(k.startswith("text_model.") for k in state_dict) else ""
        self.w = {k[len(pfx):]: v.detach().to(dtype=torch.float16).contiguous().to(self.device)
                  for k, v in state_dict.items() if k.startswith(pfx) and v.dtype.is_floating_point}
        self.n_layers = 1 + max(int(k.split(".")[2]) for k in self.w if k.startswith("encoder.layers."))
        self.width = self.w["embeddings.token_embedding.weight"].shape[1]
        self.max_positions = self.w["embeddings.position_embedding.weight"].shape[0]

    @classmethod
    def random_init(cls, seed: int = 0, device: str = "cuda", width: int = 768, layers: int = 12, heads: int = 12,
                    mlp: int = 3072, vocab: int = 49408, positions: int = 77) -> "ClipTextB200":
        """random-init weights of the CLIP-L/14 text tower shape (no checkpoint is reachable offline)"""
        g = torch.Generator().manual_seed(seed)

        def n(*shape, std=0.02):
            return torch.randn(shape, generator=g) * std

        sd = {"embeddings.token_embedding.weight": n(vocab, width), "embeddings.position_embedding.weight": n(positions, width, std=0.01),
              "final_layer_norm.weight": torch.ones(width), "final_layer_norm.bias": torch.zeros(width)}
        for i in range(layers):
            p = f"encoder.layers.{i}."
            for name in ("q_proj", "k_proj", "v_proj", "out_proj"):
                sd[p + f"self_attn.{name}.weight"], sd[p + f"self_attn.{name}.bias"] = n(width, width), torch.zeros(width)
            sd[p + "mlp.fc1.weight"], sd[p + "mlp.fc1.bias"] = n(mlp, width), torch.zeros(mlp)
            sd[p + "mlp.fc2.weight"], sd[p + "mlp.fc2.bias"] = n(width, mlp), torch.zeros(width)
            for ln in ("layer_norm1", "layer_norm2"):
                sd[p + ln + ".weight"], sd[p + ln + ".bias"] = torch.ones(width), torch.zeros(width)
        return cls(sd, device=device, heads=heads)

    @torch.no_grad()
    def __call__(self, input_ids: torch.Tensor, **_ignored) -> T.Tuple[torch.Tensor]:
        w = self.w
        ids = input_ids.to(self.device)
        B, L = ids.shape
        if L > self.max_positions:
            raise ValueError(f"sequence length {L} exceeds the {self.max_positions} positions of the text encoder")
        C, H = self.width, self.heads
        x = (w["embeddings.token_embedding.weight"][ids] + w["embeddings.position_embedding.weight"][:L][None]).reshape(B * L, C)
        x = x.contiguous()
        pitch = (L + 7) // 8 * 8
        for i in range(self.n_layers):
            p = f"encoder.layers.{i}."
            h = ops.layer_norm(x, w[p + "layer_norm1.weight"], w[p + "layer_norm1.bias"], self.eps)
            q = ops.gemm(h, w[p + "self_attn.q_proj.weight"], bias=w[p + "self_attn.q_proj.bias"]).reshape(B, L, C)
            k = ops.gemm(h, w[p + "self_attn.k_proj.weight"], bias=w[p + "self_attn.k_proj.bias"]).reshape(B, L, C)
            vt = torch.zeros((B, 1, C, pitch), dtype=torch.float16, device=self.device)
            ops.gemm(w[p + "self_attn.v_proj.weight"], h.reshape(B, 1, L, C), bias=w[p + "self_attn.v_proj.bias"], bias_per_row=True,
                     out=vt[..., :L])                                      # V^T = W_v h^T (+ b per row): K-major operand of P.V
            o = ops.attention(q.contiguous(), k.contiguous(), vt.reshape(B, C, pitch), H, L, causal=True)
            x = ops.gemm(o.reshape(B * L, C), w[p + "self_attn.out_proj.weight"], bias=w[p + "self_attn.out_proj.bias"],
                         residual=x).reshape(B * L, C)
            h = ops.layer_norm(x, w[p + "layer_norm2.weight"], w[p + "layer_norm2.bias"], self.eps)
            f = ops.gemm(h, w[p + "mlp.fc1.weight"], bias=w[p + "mlp.fc1.bias"], act=ops.ACT_QUICK_GELU).reshape(B * L, -1)
            x = ops.gemm(f, w[p + "mlp.fc2.weight"], bias=w[p + "mlp.fc2.bias"], residual=x).reshape(B * L, C)
        out = ops.layer_norm(x, w["final_layer_norm.weight"], w["final_layer_norm.bias"], self.eps)
        return (out.reshape(B, L, C),)

    def to(self, *a, **k):
        return self

    @property
    def dtype(self):
        return torch.float16
