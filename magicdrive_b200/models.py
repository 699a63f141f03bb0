"""Drop-in modules for the two networks of the hot path, and for the VAE decoder and CLIP text encoder around it.

`UNet2DConditionModelMultiview` and `BEVControlNetModel` keep the reference's constructor kwargs, parameter names
(so `load_state_dict(reference.state_dict())` and the diffusers `save_pretrained` directories load unchanged),
`forward` signatures and return types (magicdrive/networks/unet_2d_condition_multiview.py:327-339,524-527;
magicdrive/networks/unet_addon_rawbox.py:707-724,921-932), plus the helper methods the pipeline calls
(`uncond_cam_param`, `add_uncond_to_kwargs`, `prepare`).  Their arithmetic runs in `engine.py` on the sm_90a
kernels; inputs must be CUDA tensors — there is no CPU path (ops raise).
"""
import json
import logging
import os
from collections import OrderedDict
from dataclasses import asdict, dataclass, fields
from typing import Any, Dict, List, Tuple, Union

import torch
import torch.nn as nn

from . import arch, ops
from .engine import ControlNetEngine, InceptionEngine, TextEncoderEngine, UNetEngine, VaeDecoderEngine

BF16, F32 = torch.bfloat16, torch.float32


@dataclass
class UNet2DConditionOutput:
    sample: torch.Tensor

    def __getitem__(self, i):
        return (self.sample,)[i]


@dataclass
class BEVControlNetOutput:  # magicdrive/networks/output_cls.py:8-13
    down_block_res_samples: Tuple[torch.Tensor]
    mid_block_res_sample: torch.Tensor
    encoder_hidden_states_with_cam: torch.Tensor


class _Config(dict):
    """dict with attribute access, like diffusers' FrozenDict config."""
    __getattr__ = dict.__getitem__


def _register_tree(root: nn.Module, shapes: "OrderedDict[str, tuple]", dtype=F32):
    """Create nested nn.Modules so that parameter names equal the reference checkpoint keys."""
    for key, shape in shapes.items():
        parts = key.split(".")
        mod = root
        for name in parts[:-1]:
            if name not in mod._modules:
                mod.add_module(name, nn.Module())
            mod = mod._modules[name]
        t = torch.empty(shape, dtype=dtype)
        if key in arch.BUFFER_KEYS:
            mod.register_buffer(parts[-1], t)
        else:
            mod.register_parameter(parts[-1], nn.Parameter(t, requires_grad=False))


class _B200Module(nn.Module):
    config_name = "config.json"
    _cfg_cls = None

    def _init_common(self, cfg, shapes, extra_config: Dict[str, Any]):
        self.arch_cfg = cfg
        cd = {k: (list(v) if isinstance(v, tuple) else v) for k, v in asdict(cfg).items()}
        cd.update(extra_config)
        self.config = _Config(cd)
        _register_tree(self, shapes)
        self._engine = None
        self._engine_key = None
        self._ctx_cache = {}
        self._view_shard = None  # re-applied to every engine this module builds (engines are rebuilt when weights change)

    # -- nn.Module conveniences the pipeline relies on (pipeline_utils.py:624, 664-685)
    @property
    def dtype(self):
        return next(self.parameters()).dtype

    @property
    def device(self):
        return next(self.parameters()).device

    def set_use_memory_efficient_attention_xformers(self, *a, **k):  # attention is always our fused kernel
        return None

    enable_xformers_memory_efficient_attention = set_use_memory_efficient_attention_xformers

    def load_state_dict(self, state_dict, strict=True, **kw):
        r = super().load_state_dict(state_dict, strict=strict, **kw)
        self._engine = None
        self._ctx_cache = {}
        return r

    def _apply(self, fn, *a, **k):
        r = super()._apply(fn, *a, **k)
        self._engine = None
        self._ctx_cache = {}
        return r

    def reset_parameters_synthetic(self, seed=0):
        """Deterministic non-zero weights (no checkpoint ships with the reference: pretrained/.gitkeep)."""
        shapes = OrderedDict((k, tuple(v.shape)) for k, v in self.state_dict().items())
        self.load_state_dict(arch.synthetic_state_dict(shapes, seed))
        return self

    @classmethod
    def from_pretrained(cls, path, torch_dtype=None, subfolder=None, **kw):
        """Load a diffusers `save_pretrained` directory: config.json + diffusion_pytorch_model.{safetensors,bin}
        (multiview_runner.py:233-242; utils/constants.py:22-26)."""
        if subfolder:
            path = os.path.join(path, subfolder)
        with open(os.path.join(path, cls.config_name)) as f:
            raw = json.load(f)
        model = cls(**{k: v for k, v in raw.items() if not k.startswith("_")})
        st = os.path.join(path, "diffusion_pytorch_model.safetensors")
        if os.path.exists(st):
            from safetensors.torch import load_file
            sd = load_file(st)
        else:
            sd = torch.load(os.path.join(path, "diffusion_pytorch_model.bin"), map_location="cpu", weights_only=True)
        model.load_state_dict(sd, strict=True)
        if torch_dtype is not None:
            model = model.to(torch_dtype)
        return model

    def _get_engine(self, cls_):
        dev = self.device
        if dev.type != "cuda":
            raise ops._lib.MdbError(f"{type(self).__name__} runs only on a CUDA (sm_90a) device; parameters are on {dev}")
        if self._engine is None:
            self._engine = cls_(self.arch_cfg, dict(self.state_dict()), dev)
            if self._view_shard is not None and hasattr(self._engine, "set_view_shard"):
                self._engine.set_view_shard(self._view_shard)
        return self._engine

    def set_view_shard(self, shard) -> None:
        """Split the cameras across ranks (dist.ViewShard) or None; survives engine rebuilds (load_state_dict / .to())."""
        self._view_shard = shard
        if self._engine is not None and hasattr(self._engine, "set_view_shard"):
            self._engine.set_view_shard(shard)


def _timesteps_f32(timestep, n, device):
    """unet_2d_condition_multiview.py:386-402: python number, 0-dim or (V,) tensor -> fp32 [n] on device."""
    if not torch.is_tensor(timestep):
        t = torch.tensor([timestep], dtype=F32, device=device)
    else:
        t = timestep.reshape(-1).to(device=device, dtype=F32)
    if t.numel() == 1 and n > 1:
        t = t.expand(n)
    return t.contiguous()


def _pick(cfg_cls, kwargs):
    names = {f.name for f in fields(cfg_cls)}
    known = {k: (tuple(v) if isinstance(v, list) else v) for k, v in kwargs.items() if k in names}
    extra = {k: v for k, v in kwargs.items() if k not in names}
    return known, extra


class UNet2DConditionModelMultiview(_B200Module):
    """CUDA-native stand-in for magicdrive.networks.unet_2d_condition_multiview.UNet2DConditionModelMultiview."""

    def __init__(self, **kwargs):
        super().__init__()
        known, extra = _pick(arch.UNetConfig, kwargs)
        if "neighboring_view_pair" in known and known["neighboring_view_pair"] is not None:
            known["neighboring_view_pair"] = {int(k): [int(x) for x in v] for k, v in known["neighboring_view_pair"].items()}
        elif "neighboring_view_pair" in known:
            known.pop("neighboring_view_pair")
        cfg = arch.UNetConfig(**known)
        arch.check_neighbors(cfg.neighboring_view_pair, cfg.neighboring_attn_type)
        for k, want in (("use_linear_projection", False), ("class_embed_type", None), ("addition_embed_type", None),
                        ("resnet_time_scale_shift", "default"), ("dual_cross_attention", False),
                        ("upcast_attention", False), ("center_input_sample", False), ("encoder_hid_dim", None),
                        ("crossview_attn_type", "basic"), ("only_cross_attention", False), ("act_fn", "silu")):
            if extra.get(k, want) != want:
                raise ValueError(f"UNet2DConditionModelMultiview (CUDA): unsupported config {k}={extra[k]!r}")
        self._init_common(cfg, arch.unet_param_shapes(cfg), extra)

    @classmethod
    def stock_unet(cls, **kwargs):
        """The plain diffusers UNet2DConditionModel (unet_2d_condition.py:161-505) on the same engine: no cross-view attention,
        any batch size (BASELINE.json configs[0]: 1-view SD-1.5 UNet, text-only conditioning)."""
        return cls(neighboring_view_pair={}, **kwargs)

    def engine(self) -> UNetEngine:
        return self._get_engine(UNetEngine)

    def prepare_context(self, encoder_hidden_states: torch.Tensor):
        """Project the conditioning tokens to K/V for all 16 transformer blocks (cached while the tensor is unchanged)."""
        eng = self._get_engine(UNetEngine)
        key = (encoder_hidden_states.data_ptr(), encoder_hidden_states._version, tuple(encoder_hidden_states.shape),
               encoder_hidden_states.dtype)
        hit = self._ctx_cache.get("kv")
        if hit is None or hit[0] != key:
            v, lc, cdim = encoder_hidden_states.shape
            ctx = encoder_hidden_states.reshape(v * lc, cdim)
            ctx = ops.f32_to_bf16(ctx.float().contiguous()) if ctx.dtype != BF16 else ctx.contiguous()
            hit = (key, eng.context_kv(ctx), lc, encoder_hidden_states)  # keep a ref so data_ptr is not recycled
            self._ctx_cache["kv"] = hit
        return hit[1], hit[2]

    @torch.no_grad()
    def forward(self, sample, timestep, encoder_hidden_states, class_labels=None, timestep_cond=None,
                attention_mask=None, cross_attention_kwargs=None, down_block_additional_residuals=None,
                mid_block_additional_residual=None, return_dict: bool = True):
        if attention_mask is not None or class_labels is not None or timestep_cond is not None:
            raise ValueError("attention_mask / class_labels / timestep_cond are not used by the MagicDrive path")
        eng = self._get_engine(UNetEngine)
        n, c, h, w = sample.shape
        if self.arch_cfg.multiview and n % self.arch_cfg.n_cam:
            raise ValueError(f"batch {n} is not a multiple of the {self.arch_cfg.n_cam} camera views")
        ctx_kv, lc = self.prepare_context(encoder_hidden_states)
        x = ops.pack_latents(ops.nchw_to_nhwc(sample), UNetEngine.CIN_PAD)
        t = _timesteps_f32(timestep, n, sample.device)
        down = mid = None
        if down_block_additional_residuals is not None:
            down = [ops.nchw_to_nhwc(r) for r in down_block_additional_residuals]
        if mid_block_additional_residual is not None:
            mid = ops.nchw_to_nhwc(mid_block_additional_residual)
        eps = eng.forward(x, n, h, w, t, ctx_kv, lc, down, mid)  # fp32 [n*h*w, 8], first out_channels valid
        co = self.arch_cfg.out_channels
        out = eps[:, :co].reshape(n, h, w, co).permute(0, 3, 1, 2).contiguous().to(sample.dtype)
        if not return_dict:
            return (out,)
        return UNet2DConditionOutput(sample=out)


class BEVControlNetModel(_B200Module):
    """CUDA-native stand-in for magicdrive.networks.unet_addon_rawbox.BEVControlNetModel (inference path)."""

    def __init__(self, **kwargs):
        super().__init__()
        kw = dict(kwargs)
        cep = kw.pop("cam_embedder_param", None) or {}
        bep = kw.pop("bbox_embedder_param", None) or {}
        known, extra = _pick(arch.ControlNetConfig, kw)
        if cep:
            known["cam_num_freqs"] = cep.get("num_freqs", 4)
        if bep:
            if bep.get("mode", "all-xyz") != "all-xyz" or bep.get("minmax_normalize", False):
                raise ValueError("only bbox mode 'all-xyz' without minmax_normalize (SDv1.5mv_rawbox.yaml) is implemented")
            known.update(bbox_n_classes=bep.get("n_classes", 10), bbox_class_token_dim=bep.get("class_token_dim", 768),
                         bbox_num_freqs=bep.get("embedder_num_freq", 4),
                         bbox_proj_dims=tuple(bep.get("proj_dims", (768, 512, 512, 768))))
        if known.get("conditioning_embedding_out_channels") is None:
            known.pop("conditioning_embedding_out_channels", None)
        # map embedder class (unet_addon_rawbox.py:172-181): the default BEVControlNetConditioningEmbedding built from map_size,
        # or BEVControlNetConditioningEmbeddingPlus built from map_embedder_param (configs/exp/272x736.yaml:16-22)
        mcls, mpar = extra.get("map_embedder_cls"), dict(extra.get("map_embedder_param") or {})
        if mcls is not None:
            if str(mcls).rsplit(".", 1)[-1] != "BEVControlNetConditioningEmbeddingPlus":
                raise ValueError(f"map_embedder_cls {mcls!r} is not implemented (BEVControlNetConditioningEmbedding[Plus] only)")
            if "conditioning_embedding_size" not in mpar:
                raise ValueError("BEVControlNetConditioningEmbeddingPlus needs map_embedder_param.conditioning_embedding_size")
            known["map_embedding_size"] = tuple(int(v) for v in mpar["conditioning_embedding_size"])
            known["map_size"] = tuple(mpar.get("conditioning_size", (25, 200, 200)))
            known["conditioning_embedding_out_channels"] = tuple(mpar.get("block_out_channels", (16, 32, 96, 256)))
            if mpar.get("conditioning_embedding_channels", known.get("block_out_channels", (320,))[0]) != \
                    known.get("block_out_channels", (320,))[0]:
                raise ValueError("conditioning_embedding_channels must equal block_out_channels[0]")
        if known.get("map_size") is None:
            known.pop("map_size", None)
        cfg = arch.ControlNetConfig(**known)
        extra.update(cam_embedder_param=cep, bbox_embedder_param=bep,
                     controlnet_conditioning_channel_order=extra.get("controlnet_conditioning_channel_order", "rgb"),
                     global_pool_conditions=extra.get("global_pool_conditions", False))
        self._init_common(cfg, arch.controlnet_param_shapes(cfg), extra)
        # unconditional BEV map (unet_addon_rawbox.py:188-202): present (and a checkpoint key) only when configured
        um = extra.get("use_uncond_map")
        if um is not None and extra.get("drop_cond_ratio", 0.0) > 0:
            if um not in ("negative1", "random", "learnable"):
                raise TypeError(f"Unknown map type: {um}.")
            t = -torch.ones(tuple(cfg.map_size)) if um == "negative1" else torch.randn(tuple(cfg.map_size))
            if um == "learnable":
                self.register_parameter("uncond_map", nn.Parameter(t, requires_grad=False))
            else:
                self.register_buffer("uncond_map", t)
        else:
            self.uncond_map = None
        self.training = False

    def engine(self) -> ControlNetEngine:
        return self._get_engine(ControlNetEngine)

    # ---------------------------------------------------------------- helpers the pipeline calls
    def uncond_cam_param(self, repeat_size: Union[List[int], int] = 1):
        """unet_addon_rawbox.py:307-315."""
        if isinstance(repeat_size, int):
            repeat_size = [1, repeat_size]
        w = self.uncond_cam.weight[0]
        n = 1
        for r in repeat_size:
            n *= int(r)
        return w[None].expand(n, -1).reshape(*repeat_size, -1, self.arch_cfg.uncond_cam_in_dim[1])

    def add_uncond_to_kwargs(self, camera_param, bboxes_3d_data, image, max_len=None, **kwargs):
        """unet_addon_rawbox.py:625-682: uncond (null camera, zero boxes + masks) in front, cond in the tail."""
        batch_size, n_cam = camera_param.shape[:2]
        ret = dict()
        ret["camera_param"] = torch.cat([self.uncond_cam_param([batch_size, n_cam]).to(camera_param), camera_param])
        if bboxes_3d_data is None:
            if not getattr(self, "_warned_no_boxes", False):  # the reference logs this on every call; once is enough
                logging.warning("Your 'bboxes_3d_data' should not be None. If this warning keeps popping, please check your code.")
                self._warned_no_boxes = True
            if max_len is not None:
                dev = camera_param.device
                ret["bboxes_3d_data"] = {
                    "bboxes": torch.zeros([batch_size * 2, n_cam, max_len, 8, 3], device=dev),
                    "classes": torch.zeros([batch_size * 2, n_cam, max_len], device=dev, dtype=torch.long),
                    "masks": torch.zeros([batch_size * 2, n_cam, max_len], device=dev, dtype=torch.bool)}
            else:
                ret["bboxes_3d_data"] = None
        else:
            ret["bboxes_3d_data"] = dict()
            for key in ["bboxes", "classes", "masks"]:
                v = torch.cat([torch.zeros_like(bboxes_3d_data[key]), bboxes_3d_data[key]])
                if max_len is not None:
                    token_num = max_len - v.shape[2]
                    assert token_num >= 0
                    pad = torch.zeros_like(v[:, :, :1]).expand(-1, -1, token_num, *v.shape[3:])
                    v = torch.cat([v, pad], dim=2)
                ret["bboxes_3d_data"][key] = v
        # the unconditional half sees the configured uncond map instead of the scene's (substitute_with_uncond_map, :378-395)
        ret["image"] = image if self.uncond_map is None else self.uncond_map[None].expand_as(image).to(image).clone()
        for k, v in kwargs.items():
            ret[k] = v
        return ret

    @torch.no_grad()
    def prepare(self, cfg, **kwargs):
        """BEVControlNetModel.prepare -> ContinuousBBoxWithTextEmbedding.prepare / set_category_token
        (unet_addon_rawbox.py:704-705, bbox_embedder.py:117-136): with `use_text_encoder_init` the class tokens are the
        pooled CLIP embeddings of the dataset's class names (done once before training; checkpoints already carry them)."""
        if not self.config["bbox_embedder_param"].get("use_text_encoder_init", False):
            return
        tokenizer, text_encoder = kwargs["tokenizer"], kwargs["text_encoder"]
        tokens = self.bbox_embedder._class_tokens
        for idx, name in enumerate(cfg.dataset.object_classes):
            ids = tokenizer([name], padding="do_not_pad", return_tensors="pt").input_ids.to(tokens.device)
            tokens[idx].copy_(text_encoder(ids).pooler_output[0])
        self._engine = None  # weights changed: repack on the next use
        self._ctx_cache = {}

    # ---------------------------------------------------------------- step-invariant conditioning (cached)
    def _key(self, *ts):
        k = []
        for t in ts:
            if t is None:
                k.append(None)
            elif isinstance(t, dict):
                k.append(tuple((n, v.data_ptr(), v._version, tuple(v.shape)) for n, v in sorted(t.items())))
            else:
                k.append((t.data_ptr(), t._version, tuple(t.shape), t.dtype))
        return tuple(k)

    def prepare_conditions(self, camera_param, bboxes_3d_data, encoder_hidden_states, controlnet_cond):
        """Camera / box / text tokens, their K/V projections for the 7 ControlNet transformers and the BEV-map
        embedding: all independent of the latents and of the timestep, so computed once and reused across steps."""
        eng = self._get_engine(ControlNetEngine)
        key = self._key(camera_param, bboxes_3d_data, encoder_hidden_states, controlnet_cond)
        hit = self._ctx_cache.get("cond")
        if hit is None or hit[0] != key:
            n_cam = camera_param.shape[1]
            ctx = eng.context(camera_param, bboxes_3d_data, encoder_hidden_states)  # fp32 (V, Lc, 768)
            ctx_bf = ops.f32_to_bf16(ctx.reshape(-1, ctx.shape[-1]))
            kv = eng.context_kv(ctx_bf)
            memb = eng.map_embedding(controlnet_cond)  # [b, h, w, 320]
            memb = memb.repeat_interleave(n_cam, dim=0).contiguous()  # 'b ... -> (b repeat) ...' (:842-843)
            hit = (key, dict(ctx=ctx, kv=kv, lc=ctx.shape[1], map=memb),
                   (camera_param, bboxes_3d_data, encoder_hidden_states, controlnet_cond))
            self._ctx_cache["cond"] = hit
        return hit[1]

    @torch.no_grad()
    def forward(self, sample, timestep, camera_param, bboxes_3d_data, encoder_hidden_states, controlnet_cond,
                encoder_hidden_states_uncond=None, conditioning_scale: float = 1.0, class_labels=None,
                timestep_cond=None, attention_mask=None, cross_attention_kwargs=None, guess_mode: bool = False,
                return_dict: bool = True, **kwargs):
        # guess_mode: the 12 + 1 residuals are scaled by torch.logspace(-1, 0, 13) * conditioning_scale instead of one factor
        # (unet_addon_rawbox.py:897-905).  Only the MODULE-level switch exists here: the reference pipeline's guess_mode + CFG
        # branch calls add_uncond_to_emb, which has a latent bug (:684-702), so the denoiser does not offer it.
        if self.config.get("controlnet_conditioning_channel_order", "rgb") != "rgb":
            raise ValueError("only 'rgb' controlnet_conditioning_channel_order is supported")
        eng = self._get_engine(ControlNetEngine)
        b, n_cam, c, h, w = sample.shape
        cond = self.prepare_conditions(camera_param, bboxes_3d_data, encoder_hidden_states, controlnet_cond)
        x = ops.pack_latents(ops.nchw_to_nhwc(sample.reshape(b * n_cam, c, h, w)), ControlNetEngine.CIN_PAD)
        t = _timesteps_f32(timestep, b, sample.device)
        if t.numel() == b and n_cam > 1:
            t = t.repeat_interleave(n_cam)  # 'b ... -> (b repeat) ...' (:840-841)
        n_res = len(arch.controlnet_residual_channels(self.arch_cfg)) + 1  # 12 down residuals + mid
        scale = ([float(v) * float(conditioning_scale) for v in torch.logspace(-1, 0, n_res)] if guess_mode
                 else float(conditioning_scale))
        down, mid, skips, xm = eng.forward(x, b * n_cam, h, w, t, cond["kv"], cond["lc"], cond["map"], scale)
        dt = sample.dtype
        down_nchw = [ops.nhwc_to_nchw(d, s.n, s.c, s.h, s.w, F32).to(dt) for d, s in zip(down, skips)]
        mid_nchw = ops.nhwc_to_nchw(mid, xm.n, xm.c, xm.h, xm.w, F32).to(dt)
        ctx = cond["ctx"].to(dt)
        if not return_dict:
            return (down_nchw, mid_nchw, ctx)
        return BEVControlNetOutput(down_block_res_samples=down_nchw, mid_block_res_sample=mid_nchw,
                                   encoder_hidden_states_with_cam=ctx)

    @classmethod
    def from_unet(cls, unet, **kwargs):
        """unet_addon_rawbox.py:414-475: copy the encoder configuration (and weights) of a UNet."""
        u = unet.arch_cfg
        model = cls(in_channels=u.in_channels, block_out_channels=u.block_out_channels,
                    down_block_types=u.down_block_types, layers_per_block=u.layers_per_block,
                    attention_head_dim=u.attention_head_dim, cross_attention_dim=u.cross_attention_dim,
                    norm_num_groups=u.norm_num_groups, norm_eps=u.norm_eps, **kwargs)
        own = model.state_dict()
        src = {k: v for k, v in unet.state_dict().items() if k in own and own[k].shape == v.shape}
        model.load_state_dict(src, strict=False)
        return model


class DecoderOutput:  # diffusers/models/vae.py:27-36
    def __init__(self, sample):
        self.sample = sample

    def __getitem__(self, i):
        return (self.sample,)[i]


class AutoencoderKL(_B200Module):
    """Decoder half of diffusers' AutoencoderKL (models/autoencoder_kl.py) for the pipeline's `decode_latents`
    (pipeline_bev_controlnet.py:100-112): same constructor kwargs and checkpoint key names (`decoder.*`,
    `post_quant_conv.*`; `encoder.*` / `quant_conv.*` of a full checkpoint are accepted and ignored), `.config.scaling_factor`
    and `.config.block_out_channels` as the pipeline reads them (pipeline_controlnet.py:130-179), `decode(z).sample`.
    Encoding is not on the path and raises."""

    def __init__(self, **kwargs):
        super().__init__()
        known, extra = _pick(arch.VaeConfig, dict(kwargs))
        cfg = arch.VaeConfig(**{k: (tuple(v) if isinstance(v, list) else v) for k, v in known.items()})
        if cfg.act_fn != "silu" or any(t != "UpDecoderBlock2D" for t in cfg.up_block_types):
            raise ValueError("only the SD-1.5 AutoencoderKL layout (UpDecoderBlock2D, silu) is implemented")
        self._init_common(cfg, arch.vae_decoder_param_shapes(cfg), extra)
        self.training = False

    _OLD_ATTN = {"query": "to_q", "key": "to_k", "value": "to_v", "proj_attn": "to_out.0"}  # pre-0.17 checkpoint names

    def load_state_dict(self, state_dict, strict=True, **kw):
        sd = {}
        for k, v in state_dict.items():
            if k.startswith(("encoder.", "quant_conv.")):
                continue
            parts = k.split(".")
            if "attentions" in parts and parts[-2] in self._OLD_ATTN:  # attention_processor.py:_from_deprecated_attn_block
                k = ".".join(parts[:-2] + [self._OLD_ATTN[parts[-2]], parts[-1]])
            sd[k] = v
        return super().load_state_dict(sd, strict=strict, **kw)

    use_cuda_graph = True  # decode_latents replays one captured graph per shape
    _decode_graphs: dict = {}

    def engine(self) -> VaeDecoderEngine:
        eng = self._get_engine(VaeDecoderEngine)
        if getattr(self, "_graphs_for", None) is not eng:  # weights changed -> engine rebuilt -> graphs stale
            self._decode_graphs, self._graphs_for = {}, eng
        return eng

    def encode(self, *a, **k):
        raise NotImplementedError("AutoencoderKL.encode is not on the generation path (SURVEY.md §2.1); only decode is built")

    @torch.no_grad()
    def decode(self, z: torch.Tensor, return_dict: bool = True):
        """z: (n, 4, h, w) latents already divided by scaling_factor, as the pipeline passes them -> (n, 3, 8h, 8w)."""
        n, c, h, w = z.shape
        z_nhwc = z.to(F32).permute(0, 2, 3, 1).contiguous().view(-1, c)
        img = self.engine().decode(z_nhwc, n, h, w).permute(0, 3, 1, 2).to(z.dtype)
        return DecoderOutput(img) if return_dict else (img,)

    @torch.no_grad()
    def decode_latents(self, latents: torch.Tensor) -> torch.Tensor:
        """StableDiffusionBEVControlNetPipeline.decode_latents (:100-112) on (b, n_cam, 4, h, w) latents, with the
        1/scaling_factor, image/2+0.5 and clamp folded into the first and last convolution: (b, n_cam, 8h, 8w, 3) fp32."""
        b, n_cam, c, h, w = latents.shape
        z = latents.to(self.device, F32).permute(0, 1, 3, 4, 2).contiguous().view(-1, c)
        eng = self.engine()
        run = lambda zz: eng.decode(zz, b * n_cam, h, w, scale=1.0 / self.config["scaling_factor"], to_unit_range=True)
        if not (self.use_cuda_graph and z.is_cuda):
            img = run(z)
        else:
            # the decode of a given shape is one CUDA graph on resident input / output buffers (eager once to size scratch)
            key = (id(eng), b * n_cam, h, w)
            g = self._decode_graphs.get(key)
            if g is None:
                zin = z.clone()
                run(zin)
                torch.cuda.synchronize()
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph):
                    out = run(zin)
                g = self._decode_graphs[key] = (graph, zin, out)
            graph, zin, out = g
            zin.copy_(z)
            graph.replay()
            img = out.clone()
        return img.reshape(b, n_cam, *img.shape[1:])


class CLIPTextModelOutput:  # transformers modeling_outputs.BaseModelOutputWithPooling (last_hidden_state, pooler_output)
    def __init__(self, last_hidden_state, pooler_output):
        self.last_hidden_state, self.pooler_output = last_hidden_state, pooler_output

    def __getitem__(self, i):
        return (self.last_hidden_state, self.pooler_output)[i]


class _TextConfig(_Config):
    """Attribute access like transformers' PretrainedConfig: a missing name is an AttributeError, so that the pipeline's
    `hasattr(text_encoder.config, "use_attention_mask")` (pipeline_controlnet.py:360) reads False."""

    def __getattr__(self, name):
        try:
            return self[name]
        except KeyError:
            raise AttributeError(name) from None


class CLIPTextModel(_B200Module):
    """transformers' CLIPTextModel for the pipeline's prompt encoding (pipeline_controlnet.py:365-369, 417-421, called from
    pipeline_bev_controlnet.py:272) and the box class tokens (BEVControlNetModel.prepare, bbox_embedder.py:123-135): the same
    constructor (a config or its kwargs), state-dict names (`text_model.*`; the `text_model.embeddings.position_ids` buffer
    of older checkpoints is accepted and ignored), `from_pretrained(dir, subfolder="text_encoder")` and
    `forward(input_ids)` returning `.last_hidden_state`, `.pooler_output` and `[0]`.  Runs on TextEncoderEngine; each
    (batch, length) shape replays one captured CUDA graph.  Padding attention masks are not supported (SD-1.5 sets no
    `use_attention_mask`, so the pipeline never passes one)."""

    config_name = "config.json"
    use_cuda_graph = True
    _graphs: dict = {}

    def __init__(self, config=None, **kwargs):
        super().__init__()
        if config is not None:
            kwargs = {**(config.to_dict() if hasattr(config, "to_dict") else dict(config)), **kwargs}
        known, extra = _pick(arch.ClipTextConfig, kwargs)
        cfg = arch.ClipTextConfig(**known)
        if cfg.hidden_act != "quick_gelu":
            raise ValueError(f"CLIPTextModel (CUDA): hidden_act {cfg.hidden_act!r} is not implemented (quick_gelu only)")
        if cfg.hidden_size % cfg.num_attention_heads:
            raise ValueError("hidden_size must be a multiple of num_attention_heads")
        self._init_common(cfg, arch.clip_text_param_shapes(cfg), {k: v for k, v in extra.items() if not k.startswith("_")})
        self.config = _TextConfig(self.config)
        self.training = False

    def load_state_dict(self, state_dict, strict=True, **kw):
        sd = {k: v for k, v in state_dict.items() if k != "text_model.embeddings.position_ids"}
        return super().load_state_dict(sd, strict=strict, **kw)

    @classmethod
    def from_pretrained(cls, path, subfolder=None, torch_dtype=None, **kw):
        """config.json + model.safetensors or pytorch_model.bin (a transformers `save_pretrained` directory)."""
        if subfolder:
            path = os.path.join(path, subfolder)
        with open(os.path.join(path, cls.config_name)) as f:
            model = cls(**json.load(f))
        st = os.path.join(path, "model.safetensors")
        if os.path.exists(st):
            from safetensors.torch import load_file
            sd = load_file(st)
        else:
            sd = torch.load(os.path.join(path, "pytorch_model.bin"), map_location="cpu", weights_only=True)
        model.load_state_dict(sd, strict=True)
        if torch_dtype is not None:
            model = model.to(torch_dtype)
        return model

    def engine(self) -> TextEncoderEngine:
        eng = self._get_engine(TextEncoderEngine)
        if getattr(self, "_graphs_for", None) is not eng:  # weights changed -> engine rebuilt -> graphs stale
            self._graphs, self._graphs_for = {}, eng
        return eng

    @torch.no_grad()
    def forward(self, input_ids, attention_mask=None, position_ids=None, output_attentions=None, output_hidden_states=None,
                return_dict: bool = True):
        if attention_mask is not None and bool((attention_mask == 0).any()):
            raise ValueError("CLIPTextModel (CUDA): padding attention masks are not supported")
        if position_ids is not None or output_attentions or output_hidden_states:
            raise ValueError("CLIPTextModel (CUDA): position_ids / output_attentions / output_hidden_states are not supported")
        n, L = input_ids.shape
        if L > self.arch_cfg.max_position_embeddings:
            raise ValueError(f"sequence length {L} exceeds max_position_embeddings {self.arch_cfg.max_position_embeddings}")
        eng = self.engine()
        ids = input_ids.to(self.device)
        if not (self.use_cuda_graph and ids.is_cuda):
            hidden, pooled = eng.forward(ids)
        else:
            key = (n, L, ids.dtype)
            g = self._graphs.get(key)
            if g is None:
                idin = ids.clone()
                eng.forward(idin)  # eager once: packs the weights and sizes the scratch outside the capture
                torch.cuda.synchronize()
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph):
                    out = eng.forward(idin)
                g = self._graphs[key] = (graph, idin, out)
            graph, idin, out = g
            idin.copy_(ids)
            graph.replay()
            hidden, pooled = (t.clone() for t in out)
        hidden, pooled = hidden.to(self.dtype), pooled.to(self.dtype)
        if not return_dict:
            return (hidden, pooled)
        return CLIPTextModelOutput(hidden, pooled)


class InceptionV3(nn.Module):
    """Drop-in for magicdrive.misc.inception.InceptionV3 (pytorch-fid's FID Inception, inception.py:16-163): same
    constructor kwargs, DEFAULT_BLOCK_INDEX / BLOCK_INDEX_BY_DIM, parameter names (`blocks.{i}.{j}...`) and forward(inp)
    -> list of NCHW fp32 block outputs.  The arithmetic runs in engine.InceptionEngine on the sm_90a kernels, one CUDA
    graph per input shape.  Nothing is downloaded: the module is built empty and the caller loads the weights
    (`from_pretrained(path)` for the pytorch-fid `.pth`, or load_state_dict with either naming scheme).  Only the FID
    variant exists and there is no backward."""

    DEFAULT_BLOCK_INDEX = 3
    BLOCK_INDEX_BY_DIM = {64: 0, 192: 1, 768: 2, 2048: 3}

    def __init__(self, output_blocks=(DEFAULT_BLOCK_INDEX,), resize_input=True, normalize_input=True,
                 requires_grad=False, use_fid_inception=True):
        super().__init__()
        if not use_fid_inception:
            raise ValueError("only the FID Inception (use_fid_inception=True) is implemented")
        if requires_grad:
            raise ValueError("InceptionV3 here is inference-only: requires_grad=True is not supported")
        self.resize_input, self.normalize_input = resize_input, normalize_input
        self.output_blocks = sorted(output_blocks)
        self.last_needed_block = max(output_blocks)
        assert self.last_needed_block <= 3, "Last possible output block index is 3"
        for key, shape in arch.inception_param_shapes(self.last_needed_block).items():
            parts = key.split(".")
            mod = self
            for name in parts[:-1]:
                if name not in mod._modules:
                    mod.add_module(name, nn.Module())
                mod = mod._modules[name]
            if parts[-1] == "num_batches_tracked":
                mod.register_buffer(parts[-1], torch.zeros(shape, dtype=torch.long))
            elif parts[-1] in arch.INCEPTION_BN_BUFFERS:
                mod.register_buffer(parts[-1], torch.empty(shape, dtype=F32))
            else:
                mod.register_parameter(parts[-1], nn.Parameter(torch.empty(shape, dtype=F32), requires_grad=False))
        self._engine = None
        self._graphs = {}

    use_cuda_graph = True

    @property
    def device(self):
        return next(self.parameters()).device

    def load_state_dict(self, state_dict, strict=True, **kw):
        """Accepts the reference wrapper's names and the pytorch-fid weights file's (torchvision Inception3 names such as
        `Mixed_5b.branch1x1.bn.running_var`); `fc.*` and `num_batches_tracked` are ignored."""
        tv = {name: prefix for name, (prefix, _) in arch.inception_convs(self.last_needed_block).items()}
        all_tv = {m for b in arch.INCEPTION_BLOCKS for m in b}
        sd = {}
        for k, v in state_dict.items():
            if k.startswith("fc.") or k.endswith("num_batches_tracked"):
                continue
            layer = k.rsplit(".", 2)[0]  # "<torchvision layer>.conv|bn.<tensor>"
            if layer in tv:
                k = tv[layer] + k[len(layer):]
            elif layer.split(".")[0] in all_tv:
                continue  # a layer of a block this module does not build (smaller output_blocks)
            sd[k] = v
        sd.update((k, v) for k, v in self.state_dict().items() if k.endswith("num_batches_tracked"))
        r = super().load_state_dict(sd, strict=strict, **kw)
        self._engine, self._graphs = None, {}
        return r

    def _apply(self, fn, *a, **k):
        r = super()._apply(fn, *a, **k)
        self._engine, self._graphs = None, {}
        return r

    @classmethod
    def from_pretrained(cls, path, output_blocks=(DEFAULT_BLOCK_INDEX,), **kwargs):
        """Build the module and load the pytorch-fid weights file (pt_inception-2015-12-05-6726825d.pth) from a local path."""
        model = cls(output_blocks, **kwargs)
        model.load_state_dict(torch.load(path, map_location="cpu", weights_only=True))
        return model

    def engine(self) -> InceptionEngine:
        dev = self.device
        if dev.type != "cuda":
            raise ops._lib.MdbError(f"InceptionV3 runs only on a CUDA (sm_90a) device; parameters are on {dev}")
        if self._engine is None:
            self._engine = InceptionEngine(dict(self.state_dict()), dev, self.last_needed_block)
        return self._engine

    @torch.no_grad()
    def features(self, images: torch.Tensor, nhwc: bool = False, quantize: bool = False) -> List[torch.Tensor]:
        """The forward pass on a [0, 1] batch, NCHW (n, 3, h, w) or with nhwc (n, h, w, 3), optionally rounded to the 8-bit
        levels a saved PNG holds first.  One CUDA graph per (shape, dtype, layout, rounding)."""
        eng = self.engine()
        images = images.to(self.device)
        if images.dtype not in (F32, BF16):
            images = images.float()
        run = lambda x: eng.forward(x, nhwc=nhwc, quantize=quantize, resize=self.resize_input,
                                    normalize=self.normalize_input, output_blocks=tuple(self.output_blocks))
        if not self.use_cuda_graph:
            return run(images.contiguous())
        key = (tuple(images.shape), images.dtype, nhwc, quantize)
        g = self._graphs.get(key)
        if g is None:
            xin = images.contiguous().clone()
            run(xin)  # eager once: sizes the split-K scratch and packs the weights
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                outs = run(xin)
            g = self._graphs[key] = (graph, xin, outs)
        graph, xin, outs = g
        xin.copy_(images)
        graph.replay()
        return [o.clone() for o in outs]

    def forward(self, inp: torch.Tensor) -> List[torch.Tensor]:
        """inp: (N, 3, H, W) in [0, 1] -> the selected blocks' outputs, NCHW fp32, ascending block index."""
        return self.features(inp)
