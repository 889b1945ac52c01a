"""UNet3DConditionModel: reference call surface (animatediff/models/unet.py:27-726), CUDA engine underneath.

Same constructor kwargs, same state-dict keys (SURVEY App. E), same ``forward`` signature and ``.sample`` output as
the reference class, so ``scripts/inference.py`` and ``AnimationPipeline`` can use it unchanged.  The forward pass is
not an nn.Module graph: activations live as channels-last tokens ``[B*F, H, W, C]`` in bf16 or fp16 (tensor-core mode) or
fp32 (strict mode) and every operator is a libfyc_sm90a kernel (followyourclick_b200.ops):

  ResnetBlock3D  (resnet.py:296-342)   GN(cross-frame)+SiLU -> conv3x3 [+bias +time-emb row bias] -> GN+SiLU ->
                                       conv3x3 [+bias +residual | 1x1 shortcut]
  Transformer3DModel / BasicTransformerBlock (attention.py:217-308,489-564)
                                       GN -> proj_in -> LN -> fused qkv GEMM -> flash attention -> out GEMM[+res] ->
                                       LN -> q GEMM -> cross attention (text [+IP second softmax]) -> out GEMM[+res] ->
                                       LN -> GEGLU GEMM (fused epilogue) -> GEMM[+res] -> proj_out[+res]
  VanillaTemporalModule (motion_module.py:51-283)
                                       GN -> proj_in -> 2x [LN(+PE) -> qkv GEMM -> temporal attention (strided over F,
                                       no transposes) -> out GEMM[+res]] -> LN -> GEGLU FF -> proj_out[+res]
"""
import json
import math
import os
from collections import OrderedDict
from dataclasses import dataclass

import torch

from . import ops
from .modeling import FrozenDict, ParamTreeModel, geglu_interleave


@dataclass
class UNet3DConditionOutput:
    sample: torch.Tensor


class ClipContext:
    """Everything in a UNet forward that depends only on a clip's text / image conditioning and therefore not on the DDIM step
    (SURVEY 8f row 2): the context tokens in the compute dtype (text, with the image-prompt tokens of the IP-Adapter projector
    appended), and per transformer block the cross-attention K/V projections of those tokens (and K_ip/V_ip).  The reference
    recomputes all of it in every forward (unet.py:592-594, attention.py:60-75,98-106); the engine builds it once per clip
    (``UNet3DConditionModel.prepare_context``) and the per-step forward only reads it."""

    def __init__(self, ctx, kv, kvi, ip_tokens, kx=None, kxi=None):
        self.ctx, self.kv, self.kvi, self.ip_tokens = ctx, kv, kvi, ip_tokens
        # packed operands of the tensor-core cross-attention (ops.cross_attention_tc), per block: (k_and_v [Bc, 80 | 16, heads DKP + C], V^T [Bc, C, 80 | 16])
        self.kx, self.kxi = kx or {}, kxi or {}

    def tensors(self):
        out = [self.ctx] + [self.kv[k] for k in sorted(self.kv)] + [self.kvi[k] for k in sorted(self.kvi)]
        for d in (self.kx, self.kxi):
            for k in sorted(d):
                out += list(d[k])
        return out

    def copy_(self, other):
        """refresh in place (the static buffers a captured CUDA graph reads)"""
        a, b = self.tensors(), other.tensors()
        assert len(a) == len(b) and all(x.shape == y.shape and x.dtype == y.dtype for x, y in zip(a, b))
        for x, y in zip(a, b):
            x.copy_(y)
        return self


def _as_tuple(v, n):
    return tuple(v) if isinstance(v, (tuple, list)) else (v,) * n


def unet_param_spec(cfg):
    """{state-dict key: shape} for the reference architecture described by ``cfg`` (the key contract of SURVEY App. E)."""
    spec = OrderedDict()
    boc = tuple(cfg["block_out_channels"])
    n = len(boc)
    temb = boc[0] * 4
    xd = cfg["cross_attention_dim"]
    mm = cfg["motion_module_kwargs"]
    cin = cfg["in_channels"]
    if cfg["use_first_frame_condition_concat"]:
        cin = cfg["in_channels"] * 2
    elif cfg["use_first_frame_mask_condition_concat"]:
        cin = cfg["in_channels"] * 2 + 1

    def lin(p, o, i, bias=True):
        spec[p + ".weight"] = (o, i)
        if bias:
            spec[p + ".bias"] = (o,)

    def conv(p, o, i, k):
        spec[p + ".weight"] = (o, i, k, k)
        spec[p + ".bias"] = (o,)

    def norm(p, c):
        spec[p + ".weight"] = (c,)
        spec[p + ".bias"] = (c,)

    def temb_mlp(p):
        lin(p + ".linear_1", temb, boc[0])
        lin(p + ".linear_2", temb, temb)

    def resnet(p, i, o):
        norm(p + ".norm1", i); conv(p + ".conv1", o, i, 3); lin(p + ".time_emb_proj", o, temb)
        norm(p + ".norm2", o); conv(p + ".conv2", o, o, 3)
        if i != o:
            conv(p + ".conv_shortcut", o, i, 1)

    def attn(p, c, kv_dim, ip=False):
        lin(p + ".to_q", c, c, False); lin(p + ".to_k", c, kv_dim, False); lin(p + ".to_v", c, kv_dim, False)
        lin(p + ".to_out.0", c, c)
        if ip:
            lin(p + ".to_k_ip", c, kv_dim, False); lin(p + ".to_v_ip", c, kv_dim, False)

    def ff(p, c):
        lin(p + ".net.0.proj", 8 * c, c); lin(p + ".net.2", c, 4 * c)

    def proj(p, c):             # Transformer3DModel proj_in / proj_out: Linear with use_linear_projection (SD-2.x), else a 1x1 conv
        if cfg.get("use_linear_projection", False):
            lin(p, c, c)
        else:
            conv(p, c, c, 1)

    def transformer(p, c):
        norm(p + ".norm", c); proj(p + ".proj_in", c)
        q = p + ".transformer_blocks.0"
        attn(q + ".attn1", c, c); norm(q + ".norm1", c)
        attn(q + ".attn2", c, xd, cfg["use_ip_cross_attention"]); norm(q + ".norm2", c)
        ff(q + ".ff", c); norm(q + ".norm3", c)
        proj(p + ".proj_out", c)

    def motion(p, c):
        p = p + ".temporal_transformer"
        norm(p + ".norm", c); lin(p + ".proj_in", c, c)
        for b in range(mm["num_transformer_block"]):
            q = p + f".transformer_blocks.{b}"
            for j, _ in enumerate(mm["attention_block_types"]):
                a = q + f".attention_blocks.{j}"
                attn(a, c, c)
                if mm.get("temporal_position_encoding", False):
                    spec[a + ".pos_encoder.pe"] = (1, mm["temporal_position_encoding_max_len"], c)
                if mm.get("add_temporal_lora", False):
                    for nm in ("to_q", "to_k", "to_v", "to_out"):
                        lin(a + f".{nm}_lora.down", mm["rank"], c, False); lin(a + f".{nm}_lora.up", c, mm["rank"], False)
            for j, _ in enumerate(mm["attention_block_types"]):
                norm(q + f".norms.{j}", c)
            ff(q + ".ff", c); norm(q + ".ff_norm", c)
        lin(p + ".proj_out", c, c)

    def has_motion(level, decoder):
        on = cfg["use_motion_module"] and (2 ** level) in tuple(cfg["motion_module_resolutions"])
        return on and (decoder or not cfg["motion_module_decoder_only"])

    conv("conv_in", boc[0], cin, 3)
    temb_mlp("time_embedding")
    if cfg["use_camera_motion_condition"]:
        temb_mlp("camera_motion_embedding")
    if cfg["use_fps_condition"]:
        temb_mlp("fps_embedding"); temb_mlp("motion_embedding")
    out_c = boc[0]
    for i in range(n):
        in_c, out_c = out_c, boc[i]
        p = f"down_blocks.{i}"
        for j in range(cfg["layers_per_block"]):
            resnet(f"{p}.resnets.{j}", in_c if j == 0 else out_c, out_c)
            if i < n - 1:
                transformer(f"{p}.attentions.{j}", out_c)
            if has_motion(i, False):
                motion(f"{p}.motion_modules.{j}", out_c)
        if i < n - 1:
            conv(f"{p}.downsamplers.0.conv", out_c, out_c, 3)
    resnet("mid_block.resnets.0", boc[-1], boc[-1]); transformer("mid_block.attentions.0", boc[-1])
    if cfg["use_motion_module"] and cfg["motion_module_mid_block"]:
        motion("mid_block.motion_modules.0", boc[-1])
    resnet("mid_block.resnets.1", boc[-1], boc[-1])
    rev = boc[::-1]
    out_c = rev[0]
    for i in range(n):
        prev, out_c, in_c = out_c, rev[i], rev[min(i + 1, n - 1)]
        p = f"up_blocks.{i}"
        nl = cfg["layers_per_block"] + 1
        for j in range(nl):
            skip = in_c if j == nl - 1 else out_c
            resnet(f"{p}.resnets.{j}", (prev if j == 0 else out_c) + skip, out_c)
            if i > 0:
                transformer(f"{p}.attentions.{j}", out_c)
            if has_motion(n - 1 - i, True):
                motion(f"{p}.motion_modules.{j}", out_c)
        if i < n - 1:
            conv(f"{p}.upsamplers.0.conv", out_c, out_c, 3)
    norm("conv_norm_out", boc[0]); conv("conv_out", cfg["out_channels"], boc[0], 3)
    return spec


def sinusoidal_pe(max_len, d_model):
    """motion_module.py:295-299 (same torch ops, so the buffer is bit-identical to the reference's)."""
    position = torch.arange(max_len).unsqueeze(1)
    div_term = torch.exp(torch.arange(0, d_model, 2) * (-math.log(10000.0) / d_model))
    pe = torch.zeros(1, max_len, d_model)
    pe[0, :, 0::2] = torch.sin(position * div_term)
    pe[0, :, 1::2] = torch.cos(position * div_term)
    return pe


class ImageProjModel(ParamTreeModel):
    """ip_adapter/my_ip_adapter.py:28-45: Linear(clip_dim -> T*D) + LayerNorm(D); forward runs on the engine."""

    def __init__(self, cross_attention_dim=1024, clip_embeddings_dim=1024, clip_extra_context_tokens=4):
        super().__init__()
        self.cross_attention_dim, self.clip_extra_context_tokens = cross_attention_dim, clip_extra_context_tokens
        self._build_tree(OrderedDict([("proj.weight", (clip_extra_context_tokens * cross_attention_dim, clip_embeddings_dim)),
                                      ("proj.bias", (clip_extra_context_tokens * cross_attention_dim,)),
                                      ("norm.weight", (cross_attention_dim,)), ("norm.bias", (cross_attention_dim,))]))

    def forward(self, image_embeds):
        x = image_embeds.float().contiguous()
        y = ops.gemm(x, self._p("proj.weight").detach(), bias=self._p("proj.bias").detach())
        y = ops.layernorm(y.view(-1, self.cross_attention_dim), self._p("norm.weight").detach(), self._p("norm.bias").detach())
        return y.view(x.shape[0], self.clip_extra_context_tokens, self.cross_attention_dim)


class UNet3DConditionModel(ParamTreeModel):
    _supports_gradient_checkpointing = True

    def __init__(self, sample_size=None, in_channels=4, out_channels=4, center_input_sample=False, flip_sin_to_cos=True,
                 freq_shift=0,
                 down_block_types=("CrossAttnDownBlock3D", "CrossAttnDownBlock3D", "CrossAttnDownBlock3D", "DownBlock3D"),
                 mid_block_type="UNetMidBlock3DCrossAttn",
                 up_block_types=("UpBlock3D", "CrossAttnUpBlock3D", "CrossAttnUpBlock3D", "CrossAttnUpBlock3D"),
                 only_cross_attention=False, block_out_channels=(320, 640, 1280, 1280), layers_per_block=2,
                 downsample_padding=1, mid_block_scale_factor=1, act_fn="silu", norm_num_groups=32, norm_eps=1e-5,
                 cross_attention_dim=1280, attention_head_dim=8, dual_cross_attention=False, use_linear_projection=False,
                 class_embed_type=None, num_class_embeds=None, upcast_attention=False, resnet_time_scale_shift="default",
                 use_motion_module=False, motion_module_resolutions=(1, 2, 4, 8), motion_module_mid_block=False,
                 motion_module_decoder_only=False, motion_module_type=None, motion_module_kwargs=None,
                 unet_use_cross_frame_attention=None, unet_use_temporal_attention=None, use_pseudo_conv3d=False,
                 use_first_frame_condition_concat=False, image_condition_dim=1024, use_ip_cross_attention=False, scale=1.0,
                 num_tokens=4, use_camera_motion_condition=False, use_text_encoder_2=False, text_encoder_2_dim=4096,
                 use_inflated_groupnorm=False, use_fps_condition=False, use_temporal_conv=False,
                 use_first_frame_mask_condition_concat=False, **unused):
        super().__init__()
        kw = {k: v for k, v in locals().items() if k not in ("self", "unused", "__class__")}
        kw["motion_module_kwargs"] = dict(motion_module_kwargs or {})
        # use_linear_projection (SD-2.x): proj_in / proj_out of every Transformer3DModel are Linear (C, C) instead of 1x1 convs
        # (animatediff/models/attention.py:179-215,270-295) - the same GEMM on the channels-last tokens, only the key shapes differ.
        # upcast_attention (SD-2.x) makes the reference form Q K^T and the softmax in fp32 (diffusers/models/attention.py:649-660).  Every
        # engine attention kernel already does, whatever the storage dtype: the wgmma kernels (attention_tc.cu) and the mma.sync kernel
        # (attention_mma.cu) accumulate S in fp32 registers and run the softmax on them, the SIMT kernel (attention_simt.cu) and the
        # temporal kernels (temporal_mma.cu, attention_simt.cu) likewise; bf16 / fp16 is only the operand and output format.  So the flag
        # changes nothing here and is accepted as is.
        unsupported = dict(center_input_sample=False, only_cross_attention=False, dual_cross_attention=False,
                           class_embed_type=None, num_class_embeds=None, resnet_time_scale_shift="default", use_pseudo_conv3d=False,
                           use_text_encoder_2=False, use_temporal_conv=False, downsample_padding=1,
                           mid_block_scale_factor=1, act_fn="silu")
        for k, v in unsupported.items():
            if kw[k] != v:
                raise NotImplementedError(f"UNet3DConditionModel: {k}={kw[k]!r} is outside the shipped inference configs")
        if unet_use_cross_frame_attention:
            raise NotImplementedError("UNet3DConditionModel: unet_use_cross_frame_attention is not built (off in every shipped config)")
        if unet_use_temporal_attention:
            raise NotImplementedError("UNet3DConditionModel: unet_use_temporal_attention (in-block temporal attention) is not built")
        if tuple(down_block_types) != ("CrossAttnDownBlock3D",) * (len(block_out_channels) - 1) + ("DownBlock3D",):
            raise NotImplementedError(f"down_block_types {down_block_types}")
        if use_motion_module and motion_module_type != "Vanilla":
            raise ValueError(f"unknown motion_module_type {motion_module_type}")
        mm = dict(num_attention_heads=8, num_transformer_block=2, attention_block_types=("Temporal_Self", "Temporal_Self"),
                  cross_frame_attention_mode=None, temporal_position_encoding=False, temporal_position_encoding_max_len=24,
                  temporal_attention_dim_div=1, zero_initialize=True, add_temporal_lora=False, rank=4,
                  use_rope_postion_encoding=False)
        mm.update(kw["motion_module_kwargs"])
        if mm["use_rope_postion_encoding"]:
            raise NotImplementedError("UNet3DConditionModel: RoPE temporal position encoding (use_rope_postion_encoding) is not built")
        if mm["temporal_attention_dim_div"] != 1 or any(t != "Temporal_Self" for t in mm["attention_block_types"]):
            raise NotImplementedError("motion module variant outside the shipped configs")
        self._mm = mm
        self.config = FrozenDict(dict(kw, _class_name="UNet3DConditionModel", _diffusers_version="0.11.1"))
        self.sample_size = sample_size
        self.in_channels = in_channels
        self.image_proj_model = None
        cfg = dict(kw, motion_module_kwargs=mm)
        self._cfg = cfg
        spec = unet_param_spec(cfg)
        buffers = {k: sinusoidal_pe(s[1], s[2]) for k, s in spec.items() if k.endswith(".pos_encoder.pe")}
        self._build_tree(spec, buffers)
        self._heads = _as_tuple(attention_head_dim, len(block_out_channels))
        self.num_upsamplers = len(block_out_channels) - 1

    # ------------------------------------------------------------------------------------------ construction
    @classmethod
    def from_config(cls, config, **kwargs):
        cfg = {k: v for k, v in dict(config).items() if not k.startswith("_")}
        cfg.update(kwargs)
        return cls(**cfg)

    @classmethod
    def from_pretrained_2d(cls, pretrained_model_path, subfolder=None, unet_additional_kwargs=None):
        """animatediff/models/unet.py:674-726: SD-1.5 or SD-2.x 2-D UNet folder (config.json + diffusion_pytorch_model.bin)
        inflated to the 3-D model; conv_in zero-extended to 9 input channels when a concat condition is on.  An SD-2.x config's
        per-level ``attention_head_dim`` list, ``cross_attention_dim`` 1024, ``use_linear_projection`` and ``upcast_attention`` pass
        through as they are."""
        unet_additional_kwargs = dict(unet_additional_kwargs or {})
        if subfolder is not None:
            pretrained_model_path = os.path.join(pretrained_model_path, subfolder)
        config_file = os.path.join(pretrained_model_path, "config.json")
        if not os.path.isfile(config_file):
            raise RuntimeError(f"{config_file} does not exist")
        with open(config_file) as f:
            config = json.load(f)
        config["down_block_types"] = ["CrossAttnDownBlock3D"] * 3 + ["DownBlock3D"]
        config["up_block_types"] = ["UpBlock3D"] + ["CrossAttnUpBlock3D"] * 3
        model = cls.from_config(config, **unet_additional_kwargs)
        model_file = os.path.join(pretrained_model_path, "diffusion_pytorch_model.bin")
        if not os.path.isfile(model_file):
            raise RuntimeError(f"{model_file} does not exist")
        state_dict = torch.load(model_file, map_location="cpu")
        if unet_additional_kwargs.get("use_first_frame_condition_concat") or unet_additional_kwargs.get("use_first_frame_mask_condition_concat"):
            w = torch.zeros_like(model._p("conv_in.weight"))
            w[:, :4] = state_dict["conv_in.weight"]
            state_dict["conv_in.weight"] = w
        m, u = model.load_state_dict(state_dict, strict=False)
        print(f"### missing keys: {len(m)}; \n### unexpected keys: {len(u)};")
        return model

    # ------------------------------------------------------------------------------------------ packed weights
    def _fw(self, key):
        """fp32 weight (time-embedding MLPs always run in fp32)"""
        return self._cached(("fw", key), lambda: self._p(key).detach().float().contiguous())

    def _cat_w(self, name, keys, lora=None, dtype=None):
        """rows of several projections stacked (q | k | v ...), temporal LoRA merged; ``dtype`` torch.float32: the unrounded stack (the
        LN-fold packer scales it by gamma BEFORE the single rounding to the compute dtype)"""
        dt = dtype or self._compute_dtype

        def make():
            ws = []
            for i, k in enumerate(keys):
                w = self._p(k).detach().float()
                if lora is not None and self._has(lora[i] + ".down.weight"):      # motion_module.py:389-456, scale 1.0
                    w = w + self._p(lora[i] + ".up.weight").detach().float() @ self._p(lora[i] + ".down.weight").detach().float()
                ws.append(w)
            return torch.cat(ws, dim=0).to(dt).contiguous()
        return self._cached(("cat", name, dt), make)

    def _qkv_padded(self, p, heads, d, pad=64, dtype=None):
        """[Wq (heads x 64 rows, rows d..63 of every head zero) ; Wk (same) ; Wv] for the tensor-core attention kernel."""
        dt = dtype or self._compute_dtype

        def make():
            def padded(w):
                C = w.shape[1]
                wp = torch.zeros(heads, pad, C, dtype=torch.float32, device=w.device)
                wp[:, :d] = w.detach().float().view(heads, d, C)
                return wp.view(heads * pad, C)
            ws = [padded(self._p(p + ".to_q.weight")), padded(self._p(p + ".to_k.weight")), self._p(p + ".to_v.weight").detach().float()]
            return torch.cat(ws, dim=0).to(dt).contiguous()
        return self._cached(("qkvpad", p, dt), make)

    def _geglu(self, p):
        def make():
            w, b = geglu_interleave(self._p(p + ".net.0.proj.weight").detach().float(), self._p(p + ".net.0.proj.bias").detach().float())
            return w.to(self._compute_dtype).contiguous(), b
        return self._cached(("geglu", p), make)

    def _ln_fold(self, name, norm, make_w, make_bias=None, interleave=False, pe=None):
        """LayerNorm folded into its consuming GEMM (fyc.h FYC_EPI_LNFOLD):
            LN(x) W^T + b = rstd (x W"^T) + (beta W^T + b),   W" = gamma . W with every row centred (ops.ln_fold_weight).
        Returns (W" in the compute dtype, cbias = beta W^T + b in fp32[, row-bias table pe W^T for the temporal position encoding:
        (LN(x) + pe_f) W^T = LN(x) W^T + pe_f W^T]).  ``interleave``: GEGLU value / gate row interleave."""
        def make():
            w = make_w().float()                                                     # [N, K] fp32 (q/k/v stacked, padded, LoRA merged ...)
            g, b = self._p(norm + ".weight").detach().float(), self._p(norm + ".bias").detach().float()
            wp = ops.ln_fold_weight(w, g, self._compute_dtype)
            cb = w @ b
            if make_bias is not None:
                cb = cb + make_bias().float()
            rb = None
            if pe is not None:
                rb = (pe.float() @ w.t()).contiguous()                               # [max_len, N]
            if interleave:                                                           # a row permutation of W" and of the bias
                wi, cb = geglu_interleave(wp.float(), cb)
                wp = wi.to(self._compute_dtype).contiguous()
            return wp, cb.contiguous(), rb
        return self._cached(("lnfold", name), make)

    def _ln_proj(self, tok, norm, name, fold_w, plain, fold_bias=None, ok=True, geglu=False, pe=None, clips=0, frames=0, rows_per_frame=0):
        """LayerNorm `norm` of the tokens [M, C] followed by a projection.  Where the fold applies (ops.ln_fold_ok and the site's own
        condition ``ok``) the norm lives in the GEMM: one read-only statistics pass + epilogue terms (_ln_fold, cache key ``name``, built
        from the unrounded fp32 thunks ``fold_w`` / ``fold_bias``) instead of writing and re-reading a normalised copy.  Otherwise
        ops.layernorm and a plain GEMM on ``plain()`` = (packed weight, bias or None).  ``pe``: temporal position table added after the
        norm, row r belongs to frame (r // rows_per_frame) % frames of one of ``clips`` clips."""
        M, C = tok.shape
        if ops.ln_fold_ok(tok.dtype, M, C) and ok:
            w, cb, rbt = self._ln_fold(name, norm, fold_w, fold_bias, interleave=geglu, pe=pe)
            rb = None
            if pe is not None:      # (LN(x) + pe_f) W^T = LN-folded GEMM + the per-frame row-bias table pe W^T; row group = (clip, frame)
                rb = self._cached(("pe_rb", name, clips, frames), lambda: rbt[:frames].repeat(clips, 1).contiguous())
            return ops.gemm(tok, w, bias=cb, rowbias=rb, rows_per_group=rows_per_frame if pe is not None else 0, geglu=geglu,
                            ln=ops.layernorm_stats(tok))
        n = ops.layernorm(tok, self._f(norm + ".weight"), self._f(norm + ".bias"), pe=pe, rows_per_frame=rows_per_frame, frames=frames)
        w, b = plain()
        return ops.gemm(n, w, bias=b, geglu=geglu)

    @staticmethod
    def _gemm_replicas(A, rep, W, **kw):
        """``rep`` row blocks of A, each through the same GEMM (weight, bias, residual / second source shared by all of them: the CFG
        replicas over one copy of what they have in common) -> [rep * rows, N].  One replica is the plain un-sliced call."""
        if rep == 1:
            return ops.gemm(A, W, **kw)
        rows = A.shape[0] // rep
        out = torch.empty((A.shape[0], W.shape[0]), dtype=A.dtype, device=A.device)
        for r in range(rep):
            ops.gemm(A[r * rows:(r + 1) * rows], W, out=out[r * rows:(r + 1) * rows], **kw)
        return out

    def _freqs(self):
        def make():
            half = self._cfg["block_out_channels"][0] // 2
            exponent = -math.log(10000) * torch.arange(half, dtype=torch.float32) / (half - self._cfg["freq_shift"])
            return torch.exp(exponent).to(self.device)          # embeddings.py:39-44, evaluated on the host like the reference
        return self._cached(("freqs",), make)

    # ------------------------------------------------------------------------------------------ blocks
    def _gn(self, p, x, B, silu, per_frame, eps=None, groups=None, x2=None):
        eps = self._cfg["norm_eps"] if eps is None else eps
        g = self._cfg["norm_num_groups"] if groups is None else groups
        nb = x.shape[0] if (per_frame or self._cfg["use_inflated_groupnorm"]) else B
        return ops.groupnorm(x, self._f(p + ".weight"), self._f(p + ".bias"), g, eps, silu=silu, stat_batches=nb, x2=x2)

    def _temb_pack(self):
        """Every ResnetBlock3D's time_emb_proj (resnet.py:307-313) stacked into one [sum Cout, temb] fp32 matrix: the forward runs
        ONE GEMV on SiLU(emb) and each conv1 reads its column block of the [B, sum Cout] result as its row bias (fyc.h ld_rowbias)
        instead of 22 latency-bound M = 2 launches."""
        def make():
            keys = [k[:-len(".time_emb_proj.weight")] for k in self._flat_params() if k.endswith(".time_emb_proj.weight")]
            offs, o = {}, 0
            for p in keys:
                n = self._p(p + ".time_emb_proj.weight").shape[0]
                offs[p] = (o, n)
                o += n
            w = torch.cat([self._p(p + ".time_emb_proj.weight").detach().float() for p in keys], dim=0).contiguous()
            b = torch.cat([self._p(p + ".time_emb_proj.bias").detach().float() for p in keys], dim=0).contiguous()
            return w, b, offs
        return self._cached(("temb_pack",), make)

    def _resnet(self, p, x, temb_all, B, F, skip=None, temb_per_image=False):
        """``temb_per_image``: ``temb_all`` holds one row per image (use_first_frame_condition, ops.first_frame_temb_rows) instead of one
        per clip.
        ``skip``: the up blocks' `torch.cat([hidden_states, res_hidden_states], dim=1)` (unet_blocks.py:763,885) is not materialised -
        norm1 normalises [x | skip] reading both tensors in place, the 1x1 shortcut runs its K loop over the two sources.  A skip with
        fewer images than x (the conv_in output under the shared CFG prefix: ONE copy for the `rep` CFG replicas of x) is read once per
        replica instead of being duplicated."""
        NB, H, W, Cin = x.shape
        o, n = self._temb_pack()[2][p]
        temb = temb_all[:, o:o + n]                      # [B, Cout] fp32 view, row stride = sum Cout
        rep = 1 if skip is None else NB // skip.shape[0]
        if rep == 1:
            h = self._gn(p + ".norm1", x, B, True, False, x2=skip)
        else:                                            # per CFG replica: statistics are per clip, so the replicas are independent launches
            nb = NB // rep
            h = torch.empty((NB, H, W, Cin + skip.shape[-1]), dtype=x.dtype, device=x.device)
            for r in range(rep):
                ops.groupnorm(x[r * nb:(r + 1) * nb], self._f(p + ".norm1.weight"), self._f(p + ".norm1.bias"), self._cfg["norm_num_groups"],
                              self._cfg["norm_eps"], silu=True, stat_batches=nb if self._cfg["use_inflated_groupnorm"] else B // rep,
                              x2=skip, out=h[r * nb:(r + 1) * nb])
        h = ops.conv3x3(h, self._conv_w(p + ".conv1.weight"), bias=self._f(p + ".conv1.bias"), rowbias=temb,
                        images_per_group=1 if temb_per_image else F)
        h = self._gn(p + ".norm2", h, B, True, False)
        if self._has(p + ".conv_shortcut.weight"):
            w_s, b_s = self._w1x1(p + ".conv_shortcut.weight"), self._f(p + ".conv_shortcut.bias")
            res = self._gemm_replicas(x.view(-1, Cin), rep, w_s, bias=b_s, A2=None if skip is None else skip.view(-1, skip.shape[-1]))
            res = res.view(NB, H, W, -1)
        else:
            res = x if skip is None else ops.concat_channels(x, skip if rep == 1 else skip.repeat(rep, 1, 1, 1))
        return ops.conv3x3(h, self._conv_w(p + ".conv2.weight"), bias=self._f(p + ".conv2.bias"), residual=res)

    def _ff(self, p, tok, norm):
        """x + W2 (a . gelu(g)),  [a, g] = W1 LN(x) + b1  (attention.py:563, motion_module.py:282): LayerNorm `norm` folded into the GEGLU GEMM
        in tensor-core mode"""
        h = self._ln_proj(tok, norm, p + ".net.0.proj", lambda: self._p(p + ".net.0.proj.weight").detach(), lambda: self._geglu(p),
                          fold_bias=lambda: self._p(p + ".net.0.proj.bias").detach(), geglu=True,
                          ok=tok.shape[1] % 32 == 0)                 # 8 C rows in 256-row GEGLU tiles
        return ops.gemm(h, self._w(p + ".net.2.weight"), bias=self._f(p + ".net.2.bias"), residual=tok)

    def _transformer(self, p, x, ctx, heads, F, dup=1):
        """dup > 1 (shared CFG prefix, see forward_nfhwc): x holds ONE copy of the clip(s) while the context holds `dup` (uncond,
        cond); everything up to the cross-attention query is computed once, the cross-attention runs once per context replica on
        the same queries, and from its output projection on the tokens exist `dup` times.  Returns [dup * NB, H, W, C]."""
        NB, H, W, C = x.shape
        M, HW, d = NB * H * W, H * W, C // heads
        res = x.view(M, C)
        h = self._gn(p + ".norm", x, None, False, True, eps=1e-6)
        tok = ops.gemm(h.view(M, C), self._w1x1(p + ".proj_in.weight"), bias=self._f(p + ".proj_in.bias"))
        q = p + ".transformer_blocks.0"
        # self attention (attention.py:507)
        # LayerNorm -> projection pairs (norm1 -> q/k/v, norm2 -> to_q, norm3 -> GEGLU): _ln_proj
        tc_attn = ops.self_attention_tc_ok(tok.dtype, HW, d)
        pad = tc_attn and d != 64          # head dim 64: every head already is one 64-column atom, the plain [q | k | v] stack is the layout
        qkv_w = (lambda dtype=None: self._qkv_padded(q + ".attn1", heads, d, dtype=dtype)) if pad else \
            (lambda dtype=None: self._cat_w(q + ".attn1", [q + ".attn1.to_q.weight", q + ".attn1.to_k.weight", q + ".attn1.to_v.weight"], dtype=dtype))
        qkv = self._ln_proj(tok, q + ".norm1", q + ".attn1.qkv" + (".pad" if pad else ""), lambda: qkv_w(torch.float32), lambda: (qkv_w(), None))
        if tc_attn:
            # tensor-core path: q/k heads 64 columns apart (head dim 40: zero-padded by the packed weight), V transposed per image (keys contiguous)
            qkv = qkv.view(NB, HW, 2 * heads * 64 + C)
            if pad:
                ops.note_padding(2.0 * M * C * 2 * heads * (64 - d))
            vt = ops.transpose_tokens(qkv, 2 * heads * 64, C)
            o = ops.self_attention_tc(qkv, 0, heads * 64, vt, heads, d, d ** -0.5)
        elif ops.self_attention_tc80_ok(tok.dtype, HW, d):
            # head dim 80 on the tensor cores: the fused [q | k | v] buffer as the GEMM wrote it (no padding), V transposed per image
            qkv = qkv.view(NB, HW, 3 * C)
            vt = ops.transpose_tokens(qkv, 2 * C, C)
            o = ops.self_attention_tc_d80(qkv, 0, C, vt, heads, d ** -0.5)
        else:
            qkv = qkv.view(NB, HW, 3 * C)
            o = ops.attention(qkv[:, :, :C], qkv[:, :, C:2 * C], qkv[:, :, 2 * C:], heads, d ** -0.5)
        tok = ops.gemm(o.view(M, C), self._w(q + ".attn1.to_out.0.weight"), bias=self._f(q + ".attn1.to_out.0.bias"), residual=tok)
        # cross attention (attention.py:516-521; IPCrossAttention.forward :49-127); K/V of the context come from the per-clip cache
        qx = self._ln_proj(tok, q + ".norm2", q + ".attn2.to_q", lambda: self._p(q + ".attn2.to_q.weight").detach(),
                           lambda: (self._w(q + ".attn2.to_q.weight"), None)).view(NB, HW, C)
        o = torch.empty((dup * NB, HW, C), dtype=qx.dtype, device=qx.device)
        L = ctx.ctx.shape[1]
        Bq = ctx.ctx.shape[0] // dup            # clips per context replica
        ipx = self._cfg["use_ip_cross_attention"]
        for r in range(dup if p in ctx.kx else 0):       # tensor-core path (head dims 40 / 64 / 80): resident packed context, text + image keys in one launch
            T = self._cfg["num_tokens"] if ipx else 0
            sc = d ** -0.5 if (self._xformers_semantics or not ipx) else float(self._cfg["scale"])     # reference quirk, see below
            kvp, vt = (t[r * Bq:(r + 1) * Bq] for t in ctx.kx[p])
            k2 = vt2 = None
            if ipx:
                kvpi, vt2 = (t[r * Bq:(r + 1) * Bq] for t in ctx.kxi[p])
                k2 = kvpi[:, :, :heads * ops.cross_dkp(d)]
            ops.cross_attention_tc(qx, kvp[:, :, :heads * ops.cross_dkp(d)], vt, heads, d, sc, L - T, o[r * NB:(r + 1) * NB], k2=k2, vt2=vt2, Lk2=T,
                                   alpha2=float(self._cfg["scale"]), kv_batch_div=F)
        kv = ctx.kv.get(p)
        for r in range(dup if kv is not None else 0):    # one pass per context replica over the SAME queries (dup = 1: the plain case)
            o_r, kv_r = o[r * NB:(r + 1) * NB], kv[r * Bq:(r + 1) * Bq]
            if self._cfg["use_ip_cross_attention"]:
                T = self._cfg["num_tokens"]
                # reference quirk (animatediff/models/attention.py:43): without xformers the IP scale replaces d^-1/2
                sc = d ** -0.5 if self._xformers_semantics else float(self._cfg["scale"])
                kvi = ctx.kvi[p][r * Bq:(r + 1) * Bq]
                # ONE launch: text keys [:, :-T] and image keys [:, -T:] staged together, two softmaxes over the same query
                # fragments, o_text + scale * o_ip written once (attention.py:92-120)
                ops.attention(qx, kv_r[:, :L - T, :C], kv_r[:, :L - T, C:], heads, sc, out=o_r, kv_batch_div=F,
                              k2=kvi[:, L - T:, :C], v2=kvi[:, L - T:, C:], alpha2=float(self._cfg["scale"]))
            else:
                ops.attention(qx, kv_r[:, :, :C], kv_r[:, :, C:], heads, d ** -0.5, out=o_r, kv_batch_div=F)
        # the shared residual stream fans out here: same `tok` added to every replica's projection
        tok = self._gemm_replicas(o.view(dup * M, C), dup, self._w(q + ".attn2.to_out.0.weight"), bias=self._f(q + ".attn2.to_out.0.bias"), residual=tok)
        # feed forward (attention.py:563)
        tok = self._ff(q + ".ff", tok, q + ".norm3")
        out = self._gemm_replicas(tok, dup, self._w1x1(p + ".proj_out.weight"), bias=self._f(p + ".proj_out.bias"), residual=res)
        return out.view(dup * NB, H, W, C)

    def _motion(self, p, x, B, F):
        p = p + ".temporal_transformer"
        mm = self._mm
        NB, H, W, C = x.shape
        M, HW, heads = NB * H * W, H * W, mm["num_attention_heads"]
        d = C // heads
        res = x.view(M, C)
        h = self._gn(p + ".norm", x, None, False, True, eps=1e-6, groups=32)
        tok = ops.gemm(h.view(M, C), self._w(p + ".proj_in.weight"), bias=self._f(p + ".proj_in.bias"))
        for b in range(mm["num_transformer_block"]):
            q = p + f".transformer_blocks.{b}"
            for j in range(len(mm["attention_block_types"])):
                a = q + f".attention_blocks.{j}"
                pe = None
                if self._has(a + ".pos_encoder.pe"):
                    if F > self._p(a + ".pos_encoder.pe").shape[1]:
                        raise ValueError(f"video_length {F} exceeds temporal_position_encoding_max_len")
                    pe = self._cached(("pe", a), lambda a=a: self._p(a + ".pos_encoder.pe").detach()[0].float().contiguous())
                names = ["to_q", "to_k", "to_v"]
                mk = lambda dtype=None, a=a: self._cat_w(a, [a + f".{nm}.weight" for nm in names], lora=[a + f".{nm}_lora" for nm in names], dtype=dtype)
                # (LN(x) + pe_f) Wqkv^T (motion_module.py:303,378)
                qkv = self._ln_proj(tok, q + f".norms.{j}", a + ".qkv", lambda: mk(torch.float32), lambda: (mk(), None),
                                    ok=pe is None or HW % 128 == 0, pe=pe, clips=B, frames=F, rows_per_frame=HW).view(B, F, HW, 3 * C)
                o = ops.temporal_attention(qkv, heads, d ** -0.5)
                wo = self._cat_w(a + ".out", [a + ".to_out.0.weight"], lora=[a + ".to_out_lora"])
                tok = ops.gemm(o.view(M, C), wo, bias=self._f(a + ".to_out.0.bias"), residual=tok)
            tok = self._ff(q + ".ff", tok, q + ".ff_norm")
        out = ops.gemm(tok, self._w(p + ".proj_out.weight"), bias=self._f(p + ".proj_out.bias"), residual=res)
        return out.view(NB, H, W, C)

    # ------------------------------------------------------------------------------------------ forward
    def _embed(self, name, values, B, residual=None, zero_row=False):
        """``zero_row``: a timestep 0 is appended after the B rows (use_first_frame_condition, unet.py:523-524)."""
        dev = self.device
        v = torch.as_tensor(values)
        v = (v.reshape(1) if v.dim() == 0 else v.reshape(-1)).to(device=dev, dtype=torch.int64).expand(B).contiguous()
        if zero_row:
            v = torch.cat([v, torch.zeros(1, dtype=torch.int64, device=dev)])
        s = ops.timestep_embed(v, self._freqs(), self._cfg["flip_sin_to_cos"])
        h = ops.silu(ops.gemm(s, self._fw(name + ".linear_1.weight"), bias=self._f(name + ".linear_1.bias")))
        return ops.gemm(h, self._fw(name + ".linear_2.weight"), bias=self._f(name + ".linear_2.bias"), residual=residual)

    def _transformer_prefixes(self):
        cfg = self._cfg
        n = len(cfg["block_out_channels"])
        out = [f"down_blocks.{i}.attentions.{j}" for i in range(n - 1) for j in range(cfg["layers_per_block"])]
        out.append("mid_block.attentions.0")
        out += [f"up_blocks.{i}.attentions.{j}" for i in range(1, n) for j in range(cfg["layers_per_block"] + 1)]
        return out

    @torch.no_grad()
    def prepare_context(self, encoder_hidden_states, reference_images_clip_feat=None, use_ip_cross_attention=False, ip_tokens=None):
        """Per-clip, step-invariant part of the forward -> ClipContext: text tokens (b, 77, D) [+ image-prompt tokens from
        ``image_proj_model(reference_images_clip_feat)`` (unet.py:592-594), or ``ip_tokens`` if the caller already has them] in the
        compute dtype, and every transformer block's fused [K | V] (and [K_ip | V_ip]) projection of them."""
        ctx = self._to_compute(encoder_hidden_states)
        B = ctx.shape[0]
        tokens = None
        if use_ip_cross_attention:
            if ip_tokens is None:
                ipm = self.image_proj_model
                if ipm is None:
                    raise RuntimeError("use_ip_cross_attention=True but unet.image_proj_model is not set (scripts/inference.py:166)")
                ip_tokens = ipm(reference_images_clip_feat.to(self.device))
            tokens = self._to_compute(ip_tokens.float())
            ctx = ops.concat_channels(ctx.view(B, -1), tokens.view(B, -1)).view(B, -1, ctx.shape[-1])   # unet.py:592-594
        Bc, L, xd = ctx.shape
        kv, kvi, kx, kxi = {}, {}, {}, {}
        ip = self._cfg["use_ip_cross_attention"]
        T = self._cfg["num_tokens"] if ip else 0
        # tensor-core cross-attention (head dims 40 / 64 / 80): the text tokens zero-padded to 80 keys, the image tokens to 16, projected with the
        # per-head padded K weight, V transposed so that the keys are contiguous - once per clip, read by every step
        pad_t = pad_i = None
        for p in self._transformer_prefixes():
            q = p + ".transformer_blocks.0"
            C = self._p(q + ".attn2.to_q.weight").shape[0]
            heads = self._heads_of(p)
            d = C // heads
            if ops.cross_attention_tc_ok(ctx.dtype, d, L - T, T):
                if pad_t is None:
                    pad_t = torch.zeros((Bc, ops.CROSS_LK, xd), dtype=ctx.dtype, device=ctx.device)
                    pad_t[:, :L - T] = ctx[:, :L - T]
                    if ip:
                        pad_i = torch.zeros((Bc, ops.CROSS_LK2, xd), dtype=ctx.dtype, device=ctx.device)
                        pad_i[:, :T] = ctx[:, L - T:]
                kx[p] = self._cross_pack(q + ".attn2", ("to_k", "to_v"), pad_t, heads, d)
                if ip:
                    kxi[p] = self._cross_pack(q + ".attn2", ("to_k_ip", "to_v_ip"), pad_i, heads, d)
                continue
            kv[p] = ops.gemm(ctx.view(Bc * L, xd), self._cat_w(q + ".attn2", [q + ".attn2.to_k.weight", q + ".attn2.to_v.weight"])).view(Bc, L, -1)
            if ip:
                kvi[p] = ops.gemm(ctx.view(Bc * L, xd), self._cat_w(q + ".attn2ip", [q + ".attn2.to_k_ip.weight", q + ".attn2.to_v_ip.weight"])).view(Bc, L, -1)
        return ClipContext(ctx, kv, kvi, tokens, kx, kxi)

    def _heads_of(self, prefix):
        """number of heads of the transformer block at ``prefix`` (attention_head_dim is per level in this diffusers vintage)"""
        n = len(self._cfg["block_out_channels"])
        if prefix.startswith("down_blocks."):
            return self._heads[int(prefix.split(".")[1])]
        if prefix.startswith("up_blocks."):
            return self._heads[n - 1 - int(prefix.split(".")[1])]
        return self._heads[-1]

    def _cross_pack(self, a, names, ctx_pad, heads, d):
        """(k_and_v, V^T) of a zero-padded context for ops.cross_attention_tc: one GEMM with [Wk (per head padded to DKP rows) ; Wv], K a
        column view of its output, V^T [Bc, C, keys] by the token transpose."""
        dkp = ops.cross_dkp(d)
        C = heads * d

        def make():
            wk, wv = self._p(a + f".{names[0]}.weight").detach().float(), self._p(a + f".{names[1]}.weight").detach().float()
            wkp = torch.zeros(heads, dkp, wk.shape[1], dtype=torch.float32, device=wk.device)
            wkp[:, :d] = wk.view(heads, d, -1)
            return torch.cat([wkp.view(heads * dkp, -1), wv], dim=0).to(self._compute_dtype).contiguous()
        w = self._cached(("crosspack", a, names), make)
        Bc, Lp, xd = ctx_pad.shape
        kvp = ops.gemm(ctx_pad.view(Bc * Lp, xd), w).view(Bc, Lp, heads * dkp + C)
        return kvp, ops.transpose_tokens(kvp, heads * dkp, C)

    def input_channel_pad(self):
        """Channel count the engine wants for its channels-last input: 16 (zero padded) in tensor-core mode so the stem
        conv runs on the tensor cores, else the model's true input channels."""
        w = self._p("conv_in.weight")
        cin = w.shape[1]
        if cin % 8 != 0 and cin <= 16 and ops.tc_ok(self._compute_dtype, 1 << 20):
            return 16
        return cin

    _taps = None    # set to a dict to record named intermediate activations (debug / layer-wise parity)

    def _tap(self, name, x):
        if self._taps is not None:
            self._taps[name] = x.detach().float().cpu()

    def _to_compute(self, t):
        """fp32 tensor of any shape -> contiguous compute-dtype copy (conversion kernel of the engine)."""
        t = t.to(device=self.device, dtype=torch.float32).contiguous()
        if self._compute_dtype == torch.float32:
            return t
        return ops.ncfhw_to_nfhwc(t.view(1, 1, 1, 1, -1), self._compute_dtype).view(t.shape)

    def forward_nfhwc(self, x, timestep, encoder_hidden_states, fps_tensor=None, flow_control=None,
                      reference_images_clip_feat=None, camera_movement_type_tensor=None, use_ip_cross_attention=False,
                      use_camera_motion_condition=False, use_fps_condition=False, use_first_frame_condition_concat=False,
                      context=None, cfg_dup=1, use_first_frame_condition=False):
        """Engine entry: x [B, F, H, W, Cin] channels-last in the compute dtype -> fp32 [B, F, H, W, out_channels] (possibly a
        [..., :out_channels] view of a wider buffer; ops.nfhwc_to_ncfhw takes it as is).  ``context``: a ClipContext from
        ``prepare_context`` - then encoder_hidden_states / reference_images_clip_feat are not read (hoisted out of the loop).
        ``cfg_dup`` = 2 (shared CFG prefix): ``x`` holds ONE copy of the b clips although the context / fps / flow / camera tensors
        hold the CFG pair (2b rows, [uncond..., cond...]).  The reference feeds ``torch.cat([latents] * 2)`` (pipeline_animation.py:
        709), so until the first cross-attention reads the text context both halves of its batch carry identical values: conv_in, the
        first ResnetBlock3D and the first transformer's GroupNorm, proj_in, self-attention (the most expensive attention of the
        network) and query projection are computed once here and fan out at that cross-attention.  Output: [2b, F, H, W, out].
        ``use_first_frame_condition`` (unet.py:523-524, resnet.py:304-320): frame 0 of every clip gets the time embedding of t = 0, the
        other frames their clip's."""
        ops.require_cuda(x, "UNet3DConditionModel")
        cfg = self._cfg
        B, F, H, W, Cin = x.shape
        x = x.reshape(B * F, H, W, Cin)
        boc = tuple(cfg["block_out_channels"])
        n = len(boc)
        dup = int(cfg_dup)
        if dup > 1 and not (n > 1 and cfg["layers_per_block"] >= 1):
            raise ValueError("cfg_dup needs a cross-attention block at the first level")
        B = B * dup                       # batch of everything from the first cross-attention on (and of the embeddings)
        ff = bool(use_first_frame_condition)
        if ff and B > 1 and (use_camera_motion_condition or use_fps_condition):
            # unet.py:523-558: the reference adds a B-row camera / fps / motion embedding to the (B + 1)-row emb of the first-frame
            # condition, which only broadcasts for B == 1
            raise ValueError(f"use_first_frame_condition with {'use_camera_motion_condition' if use_camera_motion_condition else 'use_fps_condition'}"
                             f" needs a UNet batch of 1 (got {B}): the reference adds the {B}-row condition embedding to the {B + 1}-row time "
                             "embedding of the first-frame condition, which does not broadcast")
        ne = B + 1 if ff else B           # rows of emb: the first-frame condition appends the t = 0 row (unet.py:523-524)
        emb = self._embed("time_embedding", timestep, B, zero_row=ff)
        if use_camera_motion_condition:   # (ne = 2 rows of one value when ff: the reference's broadcast of its 1-row embedding)
            emb = self._embed("camera_motion_embedding", camera_movement_type_tensor, ne, residual=emb)
        if use_fps_condition:
            emb = self._embed("fps_embedding", fps_tensor, ne, residual=emb)
            emb = self._embed("motion_embedding", flow_control, ne, residual=emb)
        semb = ops.silu(emb)                                     # every resnet applies SiLU to emb first (resnet.py:307)
        tw, tb, _ = self._temb_pack()
        semb = ops.gemm(semb, tw, bias=tb)                       # [B, sum Cout]: all 22 time_emb_proj at once (see _temb_pack)
        if ff:                                                   # [B F, sum Cout]: frame 0 of each clip -> the t = 0 row (resnet.py:304-320)
            semb = ops.first_frame_temb_rows(semb, B, F)
        # step-invariant conditioning: built here when the caller has not hoisted it out of the DDIM loop (``context``)
        ctx = context if context is not None else self.prepare_context(
            encoder_hidden_states, reference_images_clip_feat, use_ip_cross_attention)
        if use_first_frame_condition_concat:
            w_in = self._cached(("cin_half",), lambda: (self._conv_w("conv_in.weight") * 0.5).contiguous())
            b_in = self._cached(("bin_half",), lambda: self._f("conv_in.bias") * 0.5)
        else:
            w_in, b_in = self._conv_w("conv_in.weight"), self._f("conv_in.bias")
        if Cin > w_in.shape[-1]:
            # channel-padded input (ops.build_unet_input(c_pad=16)): zero-extend the filter so the 9-channel stem takes
            # the tensor-core path (TMA needs 16-byte channel rows); the padded channels multiply zeros.
            def pad(w=w_in, c=Cin):
                wp = torch.zeros(w.shape[:-1] + (c,), dtype=w.dtype, device=w.device)
                wp[..., :w.shape[-1]] = w
                return wp
            ops.note_padding(2.0 * x.shape[0] * H * W * 9 * (Cin - w_in.shape[-1]) * w_in.shape[0])
            w_in = self._cached(("cin_pad", Cin, bool(use_first_frame_condition_concat)), pad)
        x = ops.conv3x3(x, w_in, bias=b_in)
        self._tap("conv_in", x)

        def motion_on(level, decoder):
            on = cfg["use_motion_module"] and (2 ** level) in tuple(cfg["motion_module_resolutions"])
            return on and (decoder or not cfg["motion_module_decoder_only"])

        skips = [x]
        shared = dup > 1                  # x still holds one copy per clip (rows of `semb` are identical across the CFG pair)
        for i in range(n):
            p = f"down_blocks.{i}"
            for j in range(cfg["layers_per_block"]):
                x = self._resnet(f"{p}.resnets.{j}", x, semb, B // dup if shared else B, F, temb_per_image=ff)
                if i < n - 1:
                    x = self._transformer(f"{p}.attentions.{j}", x, ctx, self._heads[i], F, dup=dup if shared else 1)
                    shared = False
                if motion_on(i, False):
                    x = self._motion(f"{p}.motion_modules.{j}", x, B, F)
                skips.append(x)
            if i < n - 1:
                x = ops.conv3x3(x, self._conv_w(f"{p}.downsamplers.0.conv.weight"), bias=self._f(f"{p}.downsamplers.0.conv.bias"), stride=2)
                skips.append(x)
            self._tap(f"down{i}", x)
        x = self._resnet("mid_block.resnets.0", x, semb, B, F, temb_per_image=ff)
        x = self._transformer("mid_block.attentions.0", x, ctx, self._heads[-1], F)
        if cfg["use_motion_module"] and cfg["motion_module_mid_block"]:
            x = self._motion("mid_block.motion_modules.0", x, B, F)
        x = self._resnet("mid_block.resnets.1", x, semb, B, F, temb_per_image=ff)
        self._tap("mid", x)
        for i in range(n):
            p = f"up_blocks.{i}"
            lvl = n - 1 - i
            for j in range(cfg["layers_per_block"] + 1):
                skip = skips.pop()                       # (under the shared CFG prefix the conv_in output exists once: _resnet reads it per replica)
                x = self._resnet(f"{p}.resnets.{j}", x, semb, B, F, skip=skip, temb_per_image=ff)
                if i > 0:
                    x = self._transformer(f"{p}.attentions.{j}", x, ctx, self._heads[lvl], F)
                if motion_on(lvl, True):
                    x = self._motion(f"{p}.motion_modules.{j}", x, B, F)
            if i < n - 1:
                x = ops.conv3x3(x, self._conv_w(f"{p}.upsamplers.0.conv.weight"), bias=self._f(f"{p}.upsamplers.0.conv.bias"), upsample=2,
                                w_phases=self._conv_w_up2(f"{p}.upsamplers.0.conv.weight"))
            self._tap(f"up{i}", x)
        x = self._gn("conv_norm_out", x, B, True, False)
        w_out, b_out, cout = self._conv_head("conv_out", x.shape[0] * H * W)
        y = ops.conv3x3(x, w_out, bias=b_out, out_f32=True)
        ops.note_padding(2.0 * x.shape[0] * H * W * 9 * x.shape[-1] * (w_out.shape[0] - cout))
        return y.view(B, F, H, W, -1)[..., :cout]          # a channel slice of the (possibly 16-wide) head output

    @torch.no_grad()
    def forward(self, sample, timestep, encoder_hidden_states, class_labels=None, attention_mask=None, return_dict=True,
                use_first_frame_condition=False, use_first_frame_condition_concat=False, use_ip_cross_attention=False,
                reference_images_latent=None, reference_images_clip_feat=None, use_camera_motion_condition=False,
                camera_movement_type_tensor=None, use_image_concat_training=False, use_text_encoder_2=False,
                encoder_hidden_states_2=None, use_fps_condition=False, fps_tensor=None, first_images_mask=None,
                flow_control=None):
        """Same signature/semantics as animatediff/models/unet.py:422-672 (sample: (b, c, f, h, w))."""
        if use_text_encoder_2 or class_labels is not None or attention_mask is not None:
            raise NotImplementedError("forward option outside the shipped inference path")
        x = sample.to(device=self.device, dtype=torch.float32)
        if use_first_frame_condition_concat and reference_images_latent is not None:          # unet.py:578-583
            first = reference_images_latent.to(x).unsqueeze(2).expand(-1, -1, x.shape[2], -1, -1)
            x = torch.cat((x, first), dim=1)
        x = ops.ncfhw_to_nfhwc(x.contiguous(), self._compute_dtype)
        y = self.forward_nfhwc(x, timestep, encoder_hidden_states, fps_tensor=fps_tensor, flow_control=flow_control,
                               reference_images_clip_feat=reference_images_clip_feat,
                               camera_movement_type_tensor=camera_movement_type_tensor,
                               use_ip_cross_attention=use_ip_cross_attention,
                               use_camera_motion_condition=use_camera_motion_condition,
                               use_fps_condition=use_fps_condition,
                               use_first_frame_condition_concat=use_first_frame_condition_concat,
                               use_first_frame_condition=use_first_frame_condition)
        out = ops.nfhwc_to_ncfhw(y)
        if not return_dict:
            return (out,)
        return UNet3DConditionOutput(sample=out)


@dataclass
class UNet2DConditionOutput:
    sample: torch.Tensor


class UNet2DConditionModel(UNet3DConditionModel):
    """Stock SD-1.5 / SD-2.x ``UNet2DConditionModel`` (diffusers/models/unet_2d_condition.py:44-439) on the engine - the T2I first-frame
    generator of scripts/inference.py:195-204,300-306 (`pipeline_base`, SURVEY 8f row 3).  It is the 3-D model without motion
    modules run on one frame: an inflated conv on F = 1 is the 2-D conv, cross-frame GroupNorm over one frame is the per-image
    GroupNorm, and the state-dict keys are the 2-D checkpoint's own (``from_pretrained_2d`` relies on exactly that).  Same
    constructor kwargs and ``forward(sample (b, 4, h, w), timestep, encoder_hidden_states).sample`` as the reference class."""

    _BLOCKS_2D_TO_3D = {"CrossAttnDownBlock2D": "CrossAttnDownBlock3D", "DownBlock2D": "DownBlock3D", "UpBlock2D": "UpBlock3D",
                        "CrossAttnUpBlock2D": "CrossAttnUpBlock3D", "UNetMidBlock2DCrossAttn": "UNetMidBlock3DCrossAttn"}

    def __init__(self, sample_size=None, in_channels=4, out_channels=4, center_input_sample=False, flip_sin_to_cos=True, freq_shift=0,
                 down_block_types=("CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "DownBlock2D"),
                 mid_block_type="UNetMidBlock2DCrossAttn",
                 up_block_types=("UpBlock2D", "CrossAttnUpBlock2D", "CrossAttnUpBlock2D", "CrossAttnUpBlock2D"),
                 only_cross_attention=False, block_out_channels=(320, 640, 1280, 1280), layers_per_block=2, downsample_padding=1,
                 mid_block_scale_factor=1, act_fn="silu", norm_num_groups=32, norm_eps=1e-5, cross_attention_dim=1280,
                 attention_head_dim=8, dual_cross_attention=False, use_linear_projection=False, class_embed_type=None,
                 num_class_embeds=None, upcast_attention=False, resnet_time_scale_shift="default"):
        m = self._BLOCKS_2D_TO_3D
        for name in tuple(down_block_types) + tuple(up_block_types) + (mid_block_type,):
            if name not in m:
                raise NotImplementedError(f"UNet2DConditionModel: block type {name}")
        super().__init__(sample_size=sample_size, in_channels=in_channels, out_channels=out_channels,
                         center_input_sample=center_input_sample, flip_sin_to_cos=flip_sin_to_cos, freq_shift=freq_shift,
                         down_block_types=tuple(m[b] for b in down_block_types), mid_block_type=m[mid_block_type],
                         up_block_types=tuple(m[b] for b in up_block_types), only_cross_attention=only_cross_attention,
                         block_out_channels=block_out_channels, layers_per_block=layers_per_block,
                         downsample_padding=downsample_padding, mid_block_scale_factor=mid_block_scale_factor, act_fn=act_fn,
                         norm_num_groups=norm_num_groups, norm_eps=norm_eps, cross_attention_dim=cross_attention_dim,
                         attention_head_dim=attention_head_dim, dual_cross_attention=dual_cross_attention,
                         use_linear_projection=use_linear_projection, class_embed_type=class_embed_type,
                         num_class_embeds=num_class_embeds, upcast_attention=upcast_attention,
                         resnet_time_scale_shift=resnet_time_scale_shift, use_motion_module=False)
        cfg2d = {k: v for k, v in locals().items() if k not in ("self", "m", "name", "__class__")}
        self.config = FrozenDict(dict(cfg2d, _class_name="UNet2DConditionModel", _diffusers_version="0.11.1"))

    @classmethod
    def from_pretrained(cls, pretrained_model_path, subfolder=None, **kwargs):
        """config.json + diffusion_pytorch_model.bin of an SD-1.5 or SD-2.x ``unet/`` folder (diffusers/modeling_utils.py:from_pretrained)."""
        if subfolder is not None:
            pretrained_model_path = os.path.join(pretrained_model_path, subfolder)
        with open(os.path.join(pretrained_model_path, "config.json")) as f:
            config = {k: v for k, v in json.load(f).items() if not k.startswith("_")}
        model = cls(**config)
        model.load_state_dict(torch.load(os.path.join(pretrained_model_path, "diffusion_pytorch_model.bin"), map_location="cpu"))
        return model

    @torch.no_grad()
    def forward(self, sample, timestep, encoder_hidden_states, class_labels=None, attention_mask=None, return_dict=True):
        if class_labels is not None or attention_mask is not None:
            raise NotImplementedError("forward option outside the SD-1.5 text-to-image path")
        out = UNet3DConditionModel.forward(self, sample.unsqueeze(2), timestep, encoder_hidden_states).sample.squeeze(2)
        if not return_dict:
            return (out,)
        return UNet2DConditionOutput(sample=out)
