"""UNetB200 — the SD-1.5 UNet2DConditionModel forward on wgmma kernels.

Drop-in at the reference's own UNet seam: `RiffusionPipeline` calls
`self.unet(latent_model_input, t, encoder_hidden_states=...)` and reads `.sample`
(riffusion/riffusion_pipeline.py:406-408); the reference itself swaps this attribute for a traced module
with exactly that duck type (`TracedUNet`, :156-169, assigned at :121).  `UNetB200.__call__` has the same
signature and returns an object with `.sample`.

Weights come from a diffusers-format state_dict (same parameter names as diffusers 0.9's
UNet2DConditionModel, see oracle/unet_oracle.py) and are repacked once: 3x3 conv kernels to
[Cout][ky][kx][Cin] (K-major for the implicit-GEMM TMA stream), everything fp16.  Activations are NHWC
fp16 end to end; the only NCHW tensors are the 4-channel latents at the two edge convolutions.

Every FLOP runs in librf_b200.so: convs and linears in the wgmma kernel (rf_conv2d_f16 /
rf_gemm_f16), norms / GEGLU / softmax in the memory-bound kernels of rf_unet_ops.cu.  No torch.nn,
cuDNN or cuBLAS call is made on this path; torch only allocates tensors and provides the stream.
"""
from __future__ import annotations

import types
import typing as T

import torch

from riffusion import tc_ops as ops


class _Out(types.SimpleNamespace):
    pass


def _h(t: torch.Tensor, device) -> torch.Tensor:
    """fp16 copy on `device`; a host tensor is converted on the host so that loading a checkpoint is memcpy only"""
    return t.detach().to(dtype=torch.float16).contiguous().to(device)


class UNetB200:
    def __init__(self, state_dict: T.Mapping[str, torch.Tensor], device: str = "cuda",
                 block_out_channels=(320, 640, 1280, 1280), heads: int = 8, groups: int = 32,
                 max_score_bytes: int = 2 << 30):
        self.device = torch.device(device)
        self.c = tuple(block_out_channels)
        self.heads, self.groups = heads, groups
        self.max_score_bytes = max_score_bytes
        self.fused_attention = True     # False: materialise fp16 scores (GEMM -> softmax -> GEMM), as the reference does
        self.fused_upsample = True      # False: nearest-2x upsample kernel + 3x3 conv, as the reference does
        self.in_channels = int(state_dict["conv_in.weight"].shape[1]) if "conv_in.weight" in state_dict else 4
        self.w: T.Dict[str, torch.Tensor] = {}
        dev = self.device
        for name, p in state_dict.items():
            if p.dim() == 4 and p.shape[2] == 3 and ".upsamplers." in name:
                self.w[name] = ops.pack_conv_weight(p.detach()).to(dev)
                self.w[name + ".up2x"] = ops.pack_upsample_weight(p.detach()).to(dev)   # four 2x2 sub-pixel phase kernels
            elif p.dim() == 4 and p.shape[2] == 3 and not name.endswith("conv_in.weight"):
                self.w[name] = ops.pack_conv_weight(p.detach()).to(dev)      # (Cout, 3, 3, Cin), packed where the tensor lives
            elif p.dim() == 4 and p.shape[2] == 1:
                self.w[name] = _h(p.reshape(p.shape[0], p.shape[1]), dev)    # 1x1 conv == linear over pixels
            elif ".ff.net.0.proj." in name:
                self.w[name] = ops.interleave_geglu(p.detach().to(torch.float16)).to(dev)   # value/gate rows paired for the epilogue
            else:
                self.w[name] = _h(p, dev)
        # all resnets' time_emb_proj (Linear 1280 -> cout) stacked into one GEMM per forward
        names = [n[: -len("time_emb_proj.weight")] for n in self.w if n.endswith("time_emb_proj.weight")]
        self._temb_slices: T.Dict[str, T.Tuple[int, int]] = {}
        if names:
            off = 0
            for n in names:
                co = self.w[n + "time_emb_proj.weight"].shape[0]
                self._temb_slices[n] = (off, off + co)
                off += co
            self._temb_w = torch.cat([self.w[n + "time_emb_proj.weight"] for n in names]).contiguous()
            self._temb_b = torch.cat([self.w[n + "time_emb_proj.bias"] for n in names]).contiguous()
        self._temb_all: T.Optional[torch.Tensor] = None

    # ------------------------------------------------------------------ building blocks
    def _resnet(self, pfx: str, x: torch.Tensor, st: T.Optional[torch.Tensor], eps: float = 1e-5,
                skip: T.Optional[torch.Tensor] = None, wrap_w: bool = False) -> torch.Tensor:
        """`skip`: the resnet's input is torch.cat([x, skip], dim=1) (up blocks); the concatenation is never materialised:
        norm1 reads both tensors in place and the 1x1 shortcut convolution takes them through its two tensor maps.
        `wrap_w`: the two 3x3 convolutions pad circularly along W."""
        w = self.w
        h = ops.group_norm(x, w[pfx + "norm1.weight"], w[pfx + "norm1.bias"], self.groups, eps, silu=True, x2=skip)
        tproj = None
        if st is not None and pfx in self._temb_slices:
            a, b = self._temb_slices[pfx]
            tproj = self._temb_all[:, a:b]
        h = ops.conv2d(h, w[pfx + "conv1.weight"], bias=w[pfx + "conv1.bias"], bias_per_image=tproj, wrap_w=wrap_w)
        h = ops.group_norm(h, w[pfx + "norm2.weight"], w[pfx + "norm2.bias"], self.groups, eps, silu=True)
        if skip is not None:                        # every concatenating resnet changes the channel count: shortcut exists
            wsc = w[pfx + "conv_shortcut.weight"]
            x = ops.conv2d(x, wsc.view(wsc.shape[0], 1, 1, wsc.shape[1]), x2=skip, bias=w[pfx + "conv_shortcut.bias"])
        elif (pfx + "conv_shortcut.weight") in w:
            B, H, W, C = x.shape
            sc = ops.gemm(x.reshape(B * H * W, C), w[pfx + "conv_shortcut.weight"], bias=w[pfx + "conv_shortcut.bias"])
            x = sc.reshape(B, H, W, -1)
        return ops.conv2d(h, w[pfx + "conv2.weight"], bias=w[pfx + "conv2.bias"], residual=x, wrap_w=wrap_w)

    def _upsample_conv(self, pfx: str, x: torch.Tensor, wrap_w: bool = False) -> torch.Tensor:
        """Upsample2D: F.interpolate(scale_factor=2, mode="nearest") then conv 3x3 pad 1 (circular along W with
        `wrap_w`)"""
        w = self.w
        if self.fused_upsample and x.shape[-1] % 64 == 0:
            return ops.conv2d_upsample2x(x, w[pfx + "weight.up2x"], bias=w[pfx + "bias"], wrap_w=wrap_w)
        return ops.conv2d(ops.upsample2x(x), w[pfx + "weight"], bias=w[pfx + "bias"], wrap_w=wrap_w)

    def _attention(self, q: torch.Tensor, k: torch.Tensor, vt: torch.Tensor, nk: int) -> torch.Tensor:
        """q: (B, Nq, C), k: (B, Nk, C), vt: (B, C, pitch>=Nk) (V transposed).  softmax(q k^T / sqrt(d)) v per head,
        scores materialised in fp16 like the reference's baddbmm/softmax/bmm (diffusers attention).  The score buffer of
        one launch stays within `max_score_bytes`: whole images per launch while one image's scores fit, else one image
        at a time in chunks of queries (a wide VAE decode)."""
        B, Nq, C = q.shape
        h = self.heads
        d = C // h
        if d <= 192 and self.fused_attention:
            return ops.attention(q.contiguous(), k.contiguous(), vt.contiguous(), h, nk)    # scores stay on the SM
        pitch = (nk + 7) // 8 * 8
        out = torch.empty((B, Nq, C), dtype=torch.float16, device=q.device)
        per_b = h * Nq * pitch * 2
        if per_b > self.max_score_bytes:
            self._attention_query_chunks(q, k, vt, nk, out)
            return out
        chunk = max(1, min(B, self.max_score_bytes // max(per_b, 1)))
        for b0 in range(0, B, chunk):
            b1 = min(B, b0 + chunk)
            qv = q[b0:b1].view(b1 - b0, Nq, h, d).permute(0, 2, 1, 3)
            kv = k[b0:b1].view(b1 - b0, nk, h, d).permute(0, 2, 1, 3)
            s = torch.empty((b1 - b0, h, Nq, pitch), dtype=torch.float16, device=q.device)
            ops.gemm(qv, kv, alpha=d ** -0.5, out=s[..., :nk])
            ops.softmax_rows_(s, nk)
            vv = vt[b0:b1].view(b1 - b0, h, d, vt.shape[-1])[..., :nk]
            ov = out[b0:b1].view(b1 - b0, Nq, h, d).permute(0, 2, 1, 3)
            ops.gemm(s[..., :nk], vv, out=ov)
        return out

    def _attention_query_chunks(self, q: torch.Tensor, k: torch.Tensor, vt: torch.Tensor, nk: int,
                                out: torch.Tensor) -> None:
        """`_attention`'s materialised path for images whose (heads, Nq, pitch) score block exceeds `max_score_bytes`:
        per image, queries in chunks of a multiple of 64 rows whose scores fit.  A query row's scores, softmax and output
        do not depend on the other rows, so only the launch shapes change."""
        B, Nq, C = q.shape
        h = self.heads
        d = C // h
        pitch = (nk + 7) // 8 * 8
        rows = max(64, self.max_score_bytes // (h * pitch * 2) // 64 * 64)
        for b in range(B):
            kv = k[b:b + 1].view(1, nk, h, d).permute(0, 2, 1, 3)
            vv = vt[b:b + 1].view(1, h, d, vt.shape[-1])[..., :nk]
            for q0 in range(0, Nq, rows):
                q1 = min(Nq, q0 + rows)
                sc = torch.empty((1, h, q1 - q0, pitch), dtype=torch.float16, device=q.device)
                qv = q[b:b + 1, q0:q1].view(1, q1 - q0, h, d).permute(0, 2, 1, 3)
                ops.gemm(qv, kv, alpha=d ** -0.5, out=sc[..., :nk])
                ops.softmax_rows_(sc, nk)
                ops.gemm(sc[..., :nk], vv, out=out[b:b + 1, q0:q1].view(1, q1 - q0, h, d).permute(0, 2, 1, 3))

    def _kv(self, pfx: str, ctx: torch.Tensor) -> T.Tuple[torch.Tensor, torch.Tensor]:
        """K = ctx Wk^T (B, Nk, C) and V^T = Wv ctx^T (B, C, pitch) — V is produced already transposed by
        swapping the GEMM operand roles, so P.V is again a K-major x K-major product."""
        w = self.w
        B, nk, cdim = ctx.shape
        k = ops.gemm(ctx.reshape(B * nk, cdim), w[pfx + "to_k.weight"]).reshape(B, nk, -1)
        C = k.shape[-1]
        pitch = (nk + 7) // 8 * 8
        vt = torch.empty((B, 1, C, pitch), dtype=torch.float16, device=ctx.device)   # columns >= nk are never read (TMA extent)
        ops.gemm(w[pfx + "to_v.weight"], ctx.unsqueeze(1), out=vt[..., :nk])
        return k, vt.reshape(B, C, pitch)

    def _transformer(self, pfx: str, x: torch.Tensor, ctx: torch.Tensor, ctx_kv) -> torch.Tensor:
        w = self.w
        B, H, W, C = x.shape
        rows = B * H * W
        h = ops.group_norm(x, w[pfx + "norm.weight"], w[pfx + "norm.bias"], self.groups, 1e-6, silu=False)
        h = ops.gemm(h.reshape(rows, C), w[pfx + "proj_in.weight"], bias=w[pfx + "proj_in.bias"]).reshape(rows, C)
        t = pfx + "transformer_blocks.0."
        # self attention
        n1 = ops.layer_norm(h, w[t + "norm1.weight"], w[t + "norm1.bias"])
        q = ops.gemm(n1, w[t + "attn1.to_q.weight"]).reshape(B, H * W, C)
        k, vt = self._kv(t + "attn1.", n1.reshape(B, H * W, C))
        o = self._attention(q, k, vt, H * W)
        h = ops.gemm(o.reshape(rows, C), w[t + "attn1.to_out.0.weight"], bias=w[t + "attn1.to_out.0.bias"],
                     residual=h).reshape(rows, C)
        # cross attention (K / V^T depend only on the text embedding: cached across denoising steps)
        n2 = ops.layer_norm(h, w[t + "norm2.weight"], w[t + "norm2.bias"])
        q = ops.gemm(n2, w[t + "attn2.to_q.weight"]).reshape(B, H * W, C)
        key = t + "attn2."
        if ctx_kv is not None and key in ctx_kv:
            k2, vt2 = ctx_kv[key]
        else:
            k2, vt2 = self._kv(key, ctx)
            if ctx_kv is not None:
                ctx_kv[key] = (k2, vt2)
        o = self._attention(q, k2, vt2, ctx.shape[1])
        h = ops.gemm(o.reshape(rows, C), w[t + "attn2.to_out.0.weight"], bias=w[t + "attn2.to_out.0.bias"],
                     residual=h).reshape(rows, C)
        # GEGLU feed-forward
        n3 = ops.layer_norm(h, w[t + "norm3.weight"], w[t + "norm3.bias"])
        g = ops.gemm(n3, w[t + "ff.net.0.proj.weight"], bias=w[t + "ff.net.0.proj.bias"],
                     act=ops.ACT_GEGLU).reshape(rows, 4 * C)                 # proj + GEGLU in the GEMM epilogue
        h = ops.gemm(g, w[t + "ff.net.2.weight"], bias=w[t + "ff.net.2.bias"], residual=h).reshape(rows, C)
        out = ops.gemm(h, w[pfx + "proj_out.weight"], bias=w[pfx + "proj_out.bias"], residual=x.reshape(rows, C))
        return out.reshape(B, H, W, C)

    # ------------------------------------------------------------------ forward
    def forward(self, sample: torch.Tensor, timestep, encoder_hidden_states: torch.Tensor,
                ctx_cache: T.Optional[dict] = None, wrap_w: bool = False) -> _Out:
        """sample: (B, 4, H, W) fp16 NCHW; timestep: int / 0-dim / (B,) tensor; encoder_hidden_states: (B, 77, 768).
        `ctx_cache`: a dict that may be reused across calls with the SAME encoder_hidden_states to skip the
        cross-attention K/V projections (they do not depend on the latents or the timestep).
        `wrap_w` (seamless loops): every 3x3 convolution pads circularly along W and with zeros along H, so the output
        tiles horizontally when the input does.  The 1x1 convolutions, norms and attention do not depend on position."""
        w = self.w
        dev = self.device
        x_in = sample.to(device=dev, dtype=torch.float16)
        ctx = encoder_hidden_states.to(device=dev, dtype=torch.float16).contiguous()
        B = x_in.shape[0]
        if torch.is_tensor(timestep) and timestep.is_cuda and timestep.dtype == torch.float32 and timestep.numel() == B:
            t = timestep
        else:
            t = torch.as_tensor(timestep, dtype=torch.float32).reshape(-1).expand(B).contiguous().to(dev)
        emb = ops.timestep_embedding(t, self.c[0])
        e1 = ops.gemm(emb, w["time_embedding.linear_1.weight"], bias=w["time_embedding.linear_1.bias"], act=ops.ACT_SILU)
        e2 = ops.gemm(e1.reshape(B, -1), w["time_embedding.linear_2.weight"], bias=w["time_embedding.linear_2.bias"])
        st = ops.silu(e2.reshape(B, -1))                       # every resnet applies SiLU to temb first
        self._temb_all = ops.gemm(st, self._temb_w, bias=self._temb_b).reshape(B, -1)

        x = ops.conv_in(x_in, w["conv_in.weight"], w["conv_in.bias"], wrap_w=wrap_w)
        skips = [x]
        n_levels = len(self.c)
        for i in range(n_levels):
            p = f"down_blocks.{i}."
            has_attn = (p + "attentions.0.norm.weight") in w
            for j in range(2):
                x = self._resnet(f"{p}resnets.{j}.", x, st, wrap_w=wrap_w)
                if has_attn:
                    x = self._transformer(f"{p}attentions.{j}.", x, ctx, ctx_cache)
                skips.append(x)
            if (p + "downsamplers.0.conv.weight") in w:
                x = ops.conv2d(x, w[p + "downsamplers.0.conv.weight"], bias=w[p + "downsamplers.0.conv.bias"], stride=2,
                               wrap_w=wrap_w)
                skips.append(x)
        x = self._resnet("mid_block.resnets.0.", x, st, wrap_w=wrap_w)
        x = self._transformer("mid_block.attentions.0.", x, ctx, ctx_cache)
        x = self._resnet("mid_block.resnets.1.", x, st, wrap_w=wrap_w)
        for i in range(n_levels):
            p = f"up_blocks.{i}."
            has_attn = (p + "attentions.0.norm.weight") in w
            for j in range(3):
                x = self._resnet(f"{p}resnets.{j}.", x, st, skip=skips.pop(), wrap_w=wrap_w)   # torch.cat([x, skip], 1) folded in
                if has_attn:
                    x = self._transformer(f"{p}attentions.{j}.", x, ctx, ctx_cache)
            if (p + "upsamplers.0.conv.weight") in w:
                x = self._upsample_conv(p + "upsamplers.0.conv.", x, wrap_w=wrap_w)
        x = ops.group_norm(x, w["conv_norm_out.weight"], w["conv_norm_out.bias"], self.groups, 1e-5, silu=True)
        out = ops.conv_out(x, w["conv_out.weight"], w["conv_out.bias"], wrap_w=wrap_w)
        return _Out(sample=out)

    def __call__(self, latent_model_input, t, encoder_hidden_states=None, **kw):
        return self.forward(latent_model_input, t, encoder_hidden_states, kw.get("ctx_cache"), kw.get("wrap_w", False))

    # diffusers-like conveniences used by pipeline code
    def to(self, *a, **k):
        return self

    @property
    def dtype(self):
        return torch.float16
