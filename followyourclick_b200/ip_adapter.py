"""IP-Adapter surface: ``IPAttnProcessor`` (ip_adapter/attention_processor.py:80-183) and ``MyIPAdapter``
(ip_adapter/my_ip_adapter.py:47-134), engine underneath.

Inside ``UNet3DConditionModel`` the same math runs as part of the fused transformer block (unet.py::_transformer,
mirroring IPCrossAttention.forward, animatediff/models/attention.py:49-127).  ``IPAttnProcessor`` is the standalone,
processor-style entry for callers that drive an attention layer themselves: identical arithmetic
``softmax(q k_text^T s) v_text + scale * softmax(q k_ip^T s) v_ip`` followed by ``to_out``, on the same kernels.
"""
from collections import OrderedDict

import torch
from torch import nn

from . import ops
from .modeling import ParamTreeModel
from .unet import ImageProjModel


class Resampler(ParamTreeModel):
    """Perceiver resampler of IP-Adapter-Plus (ip_adapter/resampler.py:87-158), engine underneath; same constructor kwargs and
    state-dict keys (``latents``, ``proj_in``, ``layers.{i}.0.{norm1,norm2,to_q,to_kv,to_out}``, ``layers.{i}.1.{0,1,3}``,
    ``proj_out``, ``norm_out``).  It is a per-clip one-off (its input, the CLIP penultimate hidden states, does not change over the
    DDIM loop - SURVEY 8f row 2), so it always runs in fp32 on the CUDA-core kernels: LayerNorm, GEMM (+bias / +residual),
    flash attention over the [image tokens ; latents] keys, exact-erf GELU - every FLOP a libfyc kernel, none in torch."""

    def __init__(self, dim=1024, depth=8, dim_head=64, heads=16, num_queries=8, embedding_dim=768, output_dim=1024, ff_mult=4,
                 max_seq_len=257, apply_pos_emb=False, num_latents_mean_pooled=0):
        super().__init__()
        if apply_pos_emb or num_latents_mean_pooled:
            raise NotImplementedError("Resampler: apply_pos_emb / num_latents_mean_pooled are off in MyIPAdapterPlus.init_proj")
        self.dim, self.depth, self.dim_head, self.heads, self.num_queries = dim, depth, dim_head, heads, num_queries
        self.embedding_dim, self.output_dim, self.ff_mult = embedding_dim, output_dim, ff_mult
        inner = dim_head * heads
        spec = OrderedDict([("latents", (1, num_queries, dim)), ("proj_in.weight", (dim, embedding_dim)), ("proj_in.bias", (dim,)),
                            ("proj_out.weight", (output_dim, dim)), ("proj_out.bias", (output_dim,)),
                            ("norm_out.weight", (output_dim,)), ("norm_out.bias", (output_dim,))])
        for i in range(depth):
            p = f"layers.{i}"
            for n in ("norm1", "norm2"):
                spec[f"{p}.0.{n}.weight"] = (dim,); spec[f"{p}.0.{n}.bias"] = (dim,)
            spec[f"{p}.0.to_q.weight"] = (inner, dim); spec[f"{p}.0.to_kv.weight"] = (2 * inner, dim)
            spec[f"{p}.0.to_out.weight"] = (dim, inner)
            spec[f"{p}.1.0.weight"] = (dim,); spec[f"{p}.1.0.bias"] = (dim,)
            spec[f"{p}.1.1.weight"] = (dim * ff_mult, dim); spec[f"{p}.1.3.weight"] = (dim, dim * ff_mult)
        self._build_tree(spec)

    @torch.no_grad()
    def forward(self, x):
        """x (b, n1, embedding_dim) -> (b, num_queries, output_dim) fp32."""
        ops.require_cuda(x, "Resampler")
        f = self._f
        B, n1, E = x.shape
        d, Q, H, inner = self.dim, self.num_queries, self.heads, self.heads * self.dim_head
        xin = ops.gemm(x.float().contiguous().view(B * n1, E), f("proj_in.weight"), bias=f("proj_in.bias"))        # [B n1, d]
        lat = f("latents").expand(B, Q, d).contiguous().view(B * Q, d)
        for i in range(self.depth):
            a, ff = f"layers.{i}.0", f"layers.{i}.1"
            xn = ops.layernorm(xin, f(a + ".norm1.weight"), f(a + ".norm1.bias"))
            ln = ops.layernorm(lat, f(a + ".norm2.weight"), f(a + ".norm2.bias"))
            q = ops.gemm(ln, f(a + ".to_q.weight")).view(B, Q, inner)
            # k, v of [x ; latents] (resampler.py:66-67): the two row blocks are projected straight into one [B, n1 + Q, 2 inner] buffer
            wkv = f(a + ".to_kv.weight").unsqueeze(0).expand(B, 2 * inner, d)
            kv = torch.empty((B, n1 + Q, 2 * inner), dtype=torch.float32, device=x.device)
            ops.gemm(xn.view(B, n1, d), wkv, out=kv[:, :n1])
            ops.gemm(ln.view(B, Q, d), wkv, out=kv[:, n1:])
            # (q s)(k s)^T with s = d_h^-1/4 (:74-75) == q k^T d_h^-1/2; softmax in fp32 (:76)
            o = ops.attention(q, kv[:, :, :inner], kv[:, :, inner:], H, self.dim_head ** -0.5)
            lat = ops.gemm(o.view(B * Q, inner), f(a + ".to_out.weight"), residual=lat)
            h = ops.layernorm(lat, f(ff + ".0.weight"), f(ff + ".0.bias"))
            h = ops.gelu(ops.gemm(h, f(ff + ".1.weight")))
            lat = ops.gemm(h, f(ff + ".3.weight"), residual=lat)
        out = ops.gemm(lat, f("proj_out.weight"), bias=f("proj_out.bias"))
        return ops.layernorm(out, f("norm_out.weight"), f("norm_out.bias")).view(B, Q, self.output_dim)


class IPAttnProcessor(nn.Module):
    def __init__(self, hidden_size, cross_attention_dim=None, scale=1.0, num_tokens=4):
        super().__init__()
        self.hidden_size, self.cross_attention_dim, self.scale, self.num_tokens = hidden_size, cross_attention_dim, scale, num_tokens
        self.to_k_ip = nn.Linear(cross_attention_dim or hidden_size, hidden_size, bias=False)
        self.to_v_ip = nn.Linear(cross_attention_dim or hidden_size, hidden_size, bias=False)
        self._compute_dtype = None          # None: fp32 / bf16 inputs run as they come, anything else in bf16

    def set_compute_dtype(self, dtype):
        """torch.float32, torch.bfloat16 or torch.float16: the dtype every call runs in, whatever the input's dtype."""
        ops.check_compute_dtype(dtype)
        self._compute_dtype = dtype
        return self

    @torch.no_grad()
    def __call__(self, attn, hidden_states, encoder_hidden_states=None, attention_mask=None, temb=None):
        """attn: object with to_q / to_k / to_v / to_out[0] (nn.Linear-like: .weight, .bias) and .heads (and optional
        .scale = d^-1/2).  hidden_states (B, L, C) or (B, C, H, W); encoder_hidden_states (B, 77+T, Dc)."""
        if attention_mask is not None:
            raise NotImplementedError("attention_mask is None on the whole inference path (SURVEY App. A.4)")
        if getattr(attn, "spatial_norm", None) is not None or getattr(attn, "group_norm", None) is not None or getattr(attn, "norm_cross", False):
            raise NotImplementedError("spatial_norm / group_norm / norm_cross are None / False for every SD-1.5 attention layer")
        ops.require_cuda(hidden_states, "IPAttnProcessor")
        nd = hidden_states.dim()
        x = hidden_states
        if nd == 4:
            b, c, h, wd = x.shape
            x = x.view(b, c, h * wd).transpose(1, 2)
        dt = self._compute_dtype or (x.dtype if x.dtype in (torch.float32, torch.bfloat16) else torch.bfloat16)
        x = x.to(dt).contiguous()
        B, Lq, C = x.shape
        heads = attn.heads
        d = C // heads
        sc = float(getattr(attn, "scale", d ** -0.5))
        w = lambda lin: lin.weight.detach().to(device=x.device, dtype=dt).contiguous()
        f = lambda t: t.detach().to(device=x.device, dtype=torch.float32).contiguous()
        q = ops.gemm(x.view(B * Lq, C), w(attn.to_q)).view(B, Lq, C)
        if encoder_hidden_states is None:
            ctx, ip = x, None
        else:
            e = encoder_hidden_states.to(device=x.device, dtype=dt).contiguous()
            end = e.shape[1] - self.num_tokens
            ctx, ip = e[:, :end].contiguous(), e[:, end:].contiguous()
        Bc, L, Dc = ctx.shape
        k = ops.gemm(ctx.view(Bc * L, Dc), w(attn.to_k)).view(Bc, L, C)
        v = ops.gemm(ctx.view(Bc * L, Dc), w(attn.to_v)).view(Bc, L, C)
        if ip is not None:           # the fused two-context kernel: text softmax + scale * image softmax, one launch, one write
            T = ip.shape[1]
            ki = ops.gemm(ip.view(Bc * T, Dc), w(self.to_k_ip)).view(Bc, T, C)
            vi = ops.gemm(ip.view(Bc * T, Dc), w(self.to_v_ip)).view(Bc, T, C)
            o = ops.attention(q, k, v, heads, sc, k2=ki, v2=vi, alpha2=float(self.scale))
        else:
            o = ops.attention(q, k, v, heads, sc)
        out_lin = attn.to_out[0]
        # residual_connection / rescale_output_factor of the modern diffusers Attention (attention_processor.py:177-180); SD-1.5 cross
        # attention has residual_connection False and factor 1
        resid = x.view(B * Lq, C) if getattr(attn, "residual_connection", False) else None
        rescale = float(getattr(attn, "rescale_output_factor", 1.0))
        if rescale != 1.0:
            raise NotImplementedError("rescale_output_factor != 1 is outside the SD-1.5 / IP-Adapter inference path")
        y = ops.gemm(o.view(B * Lq, C), w(out_lin), bias=f(out_lin.bias) if out_lin.bias is not None else None, residual=resid).view(B, Lq, C)
        if nd == 4:
            y = y.transpose(1, 2).reshape(b, c, h, wd)
        return y.to(hidden_states.dtype)


IPAttnProcessor2_0 = IPAttnProcessor


class MyIPAdapter:
    """ip_adapter/my_ip_adapter.py:47-134.  The CLIP vision tower is a per-clip one-off outside the hot path: pass any
    ``image_encoder`` callable returning ``.image_embeds`` (transformers.CLIPVisionModelWithProjection or a stub)."""

    def __init__(self, unet, image_encoder_path=None, ip_ckpt=None, device="cuda", num_tokens=4, image_encoder=None,
                 clip_embeddings_dim=None):
        self.device, self.image_encoder_path, self.ip_ckpt, self.num_tokens, self.unet = device, image_encoder_path, ip_ckpt, num_tokens, unet
        if image_encoder is None and image_encoder_path:
            from transformers import CLIPVisionModelWithProjection
            image_encoder = CLIPVisionModelWithProjection.from_pretrained(image_encoder_path).to(device)
        self.image_encoder = image_encoder
        self._clip_dim = clip_embeddings_dim or getattr(getattr(image_encoder, "config", None), "projection_dim", 1024)
        self.clip_image_processor = None
        self.image_proj_model = self.init_proj()

    def set_compute_dtype(self, dtype):
        """forwards to the UNet and the image projector (see ParamTreeModel.set_compute_dtype)"""
        ops.check_compute_dtype(dtype)
        for m in (self.unet, self.image_proj_model, getattr(self.unet, "image_proj_model", None)):
            if m is not None:
                m.set_compute_dtype(dtype)
        return self

    def init_proj(self):
        return ImageProjModel(cross_attention_dim=self.unet.config.cross_attention_dim, clip_embeddings_dim=self._clip_dim,
                              clip_extra_context_tokens=self.num_tokens).to(self.device)

    def get_ip_adapter_state_dict(self):
        """ip_adapter/my_ip_adapter.py:72-83: {"image_proj": {...}, "ip_adapter": {...}} from a .bin / .safetensors IP-Adapter file."""
        import os
        if os.path.splitext(self.ip_ckpt)[-1] == ".safetensors":
            from safetensors import safe_open
            sd = {"image_proj": {}, "ip_adapter": {}}
            with safe_open(self.ip_ckpt, framework="pt", device="cpu") as f:
                for key in f.keys():
                    for part in ("image_proj", "ip_adapter"):
                        if key.startswith(part + "."):
                            sd[part][key[len(part) + 1:]] = f.get_tensor(key)
            return sd
        return torch.load(self.ip_ckpt, map_location="cpu")

    def load_ip_adapter(self, unet=None, use_unet_image_proj_model=False, state_dict=None):
        """ip_adapter/my_ip_adapter.py:85-125 / :234-268 (load-time weight surgery, outside the hot path): the projector's weights go into
        ``unet.image_proj_model`` (or this adapter's own projector), and the adapter file's ``to_k_ip`` / ``to_v_ip`` tensors replace the
        UNet's ``*_ip*`` tensors PAIRED BY ORDER, exactly like the reference (zip of the two key lists, shapes asserted)."""
        sd = state_dict if state_dict is not None else self.get_ip_adapter_state_dict()
        target = unet if unet is not None else self.unet
        if use_unet_image_proj_model:
            if getattr(target, "image_proj_model", None) is None:
                target.image_proj_model = self.init_proj()
            target.image_proj_model.load_state_dict(sd["image_proj"])
        else:
            self.image_proj_model.load_state_dict(sd["image_proj"])
        usd = target.state_dict()
        ip_keys = list(sd["ip_adapter"].keys())
        model_keys = [k for k in usd if "_ip" in k]
        for k1, k2 in zip(model_keys, ip_keys):
            assert tuple(usd[k1].shape) == tuple(sd["ip_adapter"][k2].shape), (k1, k2)
            usd[k1] = sd["ip_adapter"][k2]
        return target.load_state_dict(usd, strict=False)

    def _pixel_values(self, input_image):
        if not torch.is_tensor(input_image):
            if self.clip_image_processor is None:
                from transformers import CLIPImageProcessor
                self.clip_image_processor = CLIPImageProcessor()
            imgs = input_image if isinstance(input_image, list) else [input_image]
            input_image = self.clip_image_processor(images=imgs, return_tensors="pt").pixel_values
        return input_image.to(self.device)

    @torch.no_grad()
    def get_image_clip_feat(self, input_image=None):
        emb = self.image_encoder(self._pixel_values(input_image)).image_embeds
        return emb, torch.zeros_like(emb)

    @torch.no_grad()
    def get_image_embeds(self, input_image=None, clip_image_embeds=None, image_proj_model=None):
        """ip_adapter/my_ip_adapter.py:136-153: (image-prompt tokens, tokens of the zero feature)."""
        if input_image is not None:
            clip_image_embeds = self.image_encoder(self._pixel_values(input_image)).image_embeds
        clip_image_embeds = clip_image_embeds.to(self.device)
        proj = image_proj_model if image_proj_model is not None else self.image_proj_model
        return proj(clip_image_embeds), proj(torch.zeros_like(clip_image_embeds))


class MyIPAdapterPlus(MyIPAdapter):
    """ip_adapter/my_ip_adapter.py:215-290: fine-grained image features - the projector is the Perceiver ``Resampler`` (depth 4,
    12 heads x 64, ``num_tokens`` queries) over the CLIP vision tower's penultimate hidden states."""

    def __init__(self, unet, image_encoder_path=None, ip_ckpt=None, device="cuda", num_tokens=16, image_encoder=None,
                 clip_embeddings_dim=None):
        super().__init__(unet, image_encoder_path, ip_ckpt, device, num_tokens, image_encoder, clip_embeddings_dim)

    def init_proj(self):
        hidden = getattr(getattr(self.image_encoder, "config", None), "hidden_size", None) or self._clip_dim
        return Resampler(dim=self.unet.config.cross_attention_dim, depth=4, dim_head=64, heads=12, num_queries=self.num_tokens,
                         embedding_dim=hidden, output_dim=self.unet.config.cross_attention_dim, ff_mult=4).to(self.device)

    @torch.no_grad()
    def get_image_clip_feat(self, input_image=None):
        input_image = self._pixel_values(input_image)
        cond = self.image_encoder(input_image, output_hidden_states=True).hidden_states[-2]
        uncond = self.image_encoder(torch.zeros_like(input_image), output_hidden_states=True).hidden_states[-2]
        return cond, uncond

    @torch.no_grad()
    def get_image_embeds(self, input_image=None, clip_image_embeds=None, image_proj_model=None):
        """ip_adapter/my_ip_adapter.py:286-305: tokens of the image's penultimate CLIP hidden states and of the zero image's."""
        cond, uncond = self.get_image_clip_feat(input_image)
        proj = image_proj_model if image_proj_model is not None else self.image_proj_model
        return proj(cond), proj(uncond)
