"""Layer enumeration of the two networks on the hot path, derived from their config alone.

Produces (a) the exact parameter names + shapes of the reference checkpoints, so our modules load
`UNet2DConditionModelMultiview` / `BEVControlNetModel` state dicts unchanged, and (b) a structural "program"
(list of resnet / transformer / sampler steps) that both the CUDA engine and the CPU oracle walk.

Reference structure: diffusers/models/unet_2d_condition.py:161-505 (constructor), unet_2d_blocks.py:794-941,
944-1027, 478-584, 1886-2030, 2033-2111; magicdrive/networks/unet_2d_condition_multiview.py:123-235;
magicdrive/networks/unet_addon_rawbox.py:33-286; bbox_embedder.py:32-108; map_embedder.py:20-64.
"""
from collections import OrderedDict
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

DEFAULT_NEIGHBORS = {0: [5, 1], 1: [0, 2], 2: [1, 3], 3: [2, 4], 4: [3, 5], 5: [4, 0]}
ATT_MAX_SETS = 8  # MDB_ATT_MAX_SETS (include/magicdrive_b200.h): neighbours one view's cross-view attention may sum


def check_neighbors(nb: Dict[int, List[int]], attn_type: str) -> None:
    """Raise ValueError, naming the view, for a camera rig the cross-view attention cannot run: the keys of
    `neighboring_view_pair` must be exactly the views 0..n_cam-1, every neighbour one of them, at most ATT_MAX_SETS
    neighbours per view, and none empty under "concat" (the reference's torch.cat of no tensors fails there too)."""
    n_cam = len(nb)
    if sorted(nb) != list(range(n_cam)):
        raise ValueError(f"neighboring_view_pair keys must be the views 0..{n_cam - 1}, got {sorted(nb)}")
    for view, values in nb.items():
        bad = [x for x in values if not 0 <= x < n_cam]
        if bad:
            raise ValueError(f"neighboring_view_pair[{view}]: neighbour(s) {bad} outside the views 0..{n_cam - 1}")
        if len(values) > ATT_MAX_SETS:
            raise ValueError(f"neighboring_view_pair[{view}] lists {len(values)} neighbours; at most {ATT_MAX_SETS} are supported")
        if not values and attn_type == "concat":
            raise ValueError(f"neighboring_view_pair[{view}] is empty: neighboring_attn_type 'concat' needs a neighbour per view")


@dataclass
class UNetConfig:
    in_channels: int = 4
    out_channels: int = 4
    block_out_channels: Tuple[int, ...] = (320, 640, 1280, 1280)
    down_block_types: Tuple[str, ...] = ("CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D",
                                         "DownBlock2D")
    up_block_types: Tuple[str, ...] = ("UpBlock2D", "CrossAttnUpBlock2D", "CrossAttnUpBlock2D", "CrossAttnUpBlock2D")
    layers_per_block: int = 2
    attention_head_dim: int = 8  # diffusers 0.17.1 passes this as the NUMBER of heads (unet_2d_blocks.py:842-845)
    cross_attention_dim: int = 768
    norm_num_groups: int = 32
    norm_eps: float = 1e-5
    flip_sin_to_cos: bool = True
    freq_shift: int = 0
    neighboring_view_pair: Dict[int, List[int]] = field(default_factory=lambda: dict(DEFAULT_NEIGHBORS))
    neighboring_attn_type: str = "add"
    zero_module_type: str = "zero_linear"
    sample_size: Optional[int] = 64

    @property
    def time_embed_dim(self):
        return self.block_out_channels[0] * 4

    @property
    def n_cam(self):
        return len(self.neighboring_view_pair)

    @property
    def multiview(self) -> bool:
        """False (no neighbouring_view_pair) = the stock diffusers UNet2DConditionModel: BasicTransformerBlock without the
        cross-view attention (BASELINE.json configs[0]: 1-view SD-1.5 UNet, text-only conditioning)."""
        return len(self.neighboring_view_pair) > 0


@dataclass
class ControlNetConfig:
    in_channels: int = 4
    block_out_channels: Tuple[int, ...] = (320, 640, 1280, 1280)
    down_block_types: Tuple[str, ...] = ("CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D",
                                         "DownBlock2D")
    layers_per_block: int = 2
    attention_head_dim: int = 8
    cross_attention_dim: int = 768
    norm_num_groups: int = 32
    norm_eps: float = 1e-5
    flip_sin_to_cos: bool = True
    freq_shift: int = 0
    # BEV specifics (configs/model/SDv1.5mv_rawbox.yaml)
    uncond_cam_in_dim: Tuple[int, int] = (3, 7)
    camera_in_dim: int = 189
    camera_out_dim: int = 768
    map_size: Tuple[int, int, int] = (8, 200, 200)
    conditioning_embedding_out_channels: Tuple[int, ...] = (16, 32, 96, 256)
    # map_embedder_cls BEVControlNetConditioningEmbeddingPlus (configs/exp/272x736.yaml:16-22): (h, w) of its AdaptiveAvgPool2d,
    # i.e. the latent grid the BEV-map embedding is pooled to; None = the plain BEVControlNetConditioningEmbedding
    map_embedding_size: Optional[Tuple[int, int]] = None
    cam_num_freqs: int = 4
    # bbox embedder (ContinuousBBoxWithTextEmbedding, mode all-xyz, minmax_normalize False)
    bbox_n_classes: int = 10
    bbox_class_token_dim: int = 768
    bbox_num_freqs: int = 4
    bbox_proj_dims: Tuple[int, ...] = (768, 512, 512, 768)
    bbox_points: int = 8

    @property
    def time_embed_dim(self):
        return self.block_out_channels[0] * 4


# ------------------------------------------------------------------------------------------ structural program
@dataclass
class ResnetSpec:
    prefix: str
    cin: int
    cout: int
    skip_c: int = 0  # channels taken from the skip connection (concatenated AFTER the running tensor)

    @property
    def shortcut(self):
        return self.cin != self.cout


@dataclass
class TransformerSpec:
    prefix: str
    c: int
    heads: int
    multiview: bool


@dataclass
class SamplerSpec:
    prefix: str
    c: int
    kind: str  # "down" (3x3 stride 2 pad 1) or "up" (nearest resize + 3x3)


@dataclass
class BlockSpec:
    name: str
    layers: List[Tuple[ResnetSpec, Optional[TransformerSpec]]]
    sampler: Optional[SamplerSpec]


def _heads(cfg, i):
    a = cfg.attention_head_dim
    return a[i] if isinstance(a, (tuple, list)) else a


def down_blocks(cfg, multiview: bool) -> List[BlockSpec]:
    blocks = []
    out_c = cfg.block_out_channels[0]
    for i, typ in enumerate(cfg.down_block_types):
        in_c, out_c = out_c, cfg.block_out_channels[i]
        final = i == len(cfg.block_out_channels) - 1
        layers = []
        for j in range(cfg.layers_per_block):
            rs = ResnetSpec(f"down_blocks.{i}.resnets.{j}", in_c if j == 0 else out_c, out_c)
            tr = None
            if typ == "CrossAttnDownBlock2D":
                tr = TransformerSpec(f"down_blocks.{i}.attentions.{j}", out_c, _heads(cfg, i), multiview)
            layers.append((rs, tr))
        samp = None if final else SamplerSpec(f"down_blocks.{i}.downsamplers.0.conv", out_c, "down")
        blocks.append(BlockSpec(f"down_blocks.{i}", layers, samp))
    return blocks


def mid_block(cfg, multiview: bool):
    c = cfg.block_out_channels[-1]
    return (ResnetSpec("mid_block.resnets.0", c, c),
            TransformerSpec("mid_block.attentions.0", c, _heads(cfg, len(cfg.block_out_channels) - 1), multiview),
            ResnetSpec("mid_block.resnets.1", c, c))


def up_blocks(cfg: UNetConfig) -> List[BlockSpec]:
    blocks = []
    rev = list(reversed(cfg.block_out_channels))
    a = cfg.attention_head_dim
    rev_heads = list(reversed(a)) if isinstance(a, (tuple, list)) else [a] * len(rev)
    out_c = rev[0]
    n = len(cfg.up_block_types)
    for i, typ in enumerate(cfg.up_block_types):
        prev_out = out_c
        out_c = rev[i]
        in_c = rev[min(i + 1, len(rev) - 1)]
        final = i == n - 1
        layers = []
        for j in range(cfg.layers_per_block + 1):
            skip_c = in_c if j == cfg.layers_per_block else out_c
            run_c = prev_out if j == 0 else out_c
            rs = ResnetSpec(f"up_blocks.{i}.resnets.{j}", run_c + skip_c, out_c, skip_c=skip_c)
            tr = None
            if typ == "CrossAttnUpBlock2D":
                tr = TransformerSpec(f"up_blocks.{i}.attentions.{j}", out_c, rev_heads[i], cfg.multiview)
            layers.append((rs, tr))
        samp = None if final else SamplerSpec(f"up_blocks.{i}.upsamplers.0.conv", out_c, "up")
        blocks.append(BlockSpec(f"up_blocks.{i}", layers, samp))
    return blocks


# ------------------------------------------------------------------------------------------ parameter shapes
def _conv(sh, p, co, ci, k, bias=True):
    sh[p + ".weight"] = (co, ci, k, k)
    if bias:
        sh[p + ".bias"] = (co,)


def _lin(sh, p, co, ci, bias=True):
    sh[p + ".weight"] = (co, ci)
    if bias:
        sh[p + ".bias"] = (co,)


def _norm(sh, p, c):
    sh[p + ".weight"] = (c,)
    sh[p + ".bias"] = (c,)


def _resnet_shapes(sh, rs: ResnetSpec, temb):
    _norm(sh, rs.prefix + ".norm1", rs.cin)
    _conv(sh, rs.prefix + ".conv1", rs.cout, rs.cin, 3)
    _lin(sh, rs.prefix + ".time_emb_proj", rs.cout, temb)
    _norm(sh, rs.prefix + ".norm2", rs.cout)
    _conv(sh, rs.prefix + ".conv2", rs.cout, rs.cout, 3)
    if rs.shortcut:
        _conv(sh, rs.prefix + ".conv_shortcut", rs.cout, rs.cin, 1)


def _attn_shapes(sh, p, c, kv):
    _lin(sh, p + ".to_q", c, c, bias=False)
    _lin(sh, p + ".to_k", c, kv, bias=False)
    _lin(sh, p + ".to_v", c, kv, bias=False)
    _lin(sh, p + ".to_out.0", c, c)


def _transformer_shapes(sh, tr: TransformerSpec, cross):
    p = tr.prefix
    _norm(sh, p + ".norm", tr.c)
    _conv(sh, p + ".proj_in", tr.c, tr.c, 1)
    b = p + ".transformer_blocks.0"
    _norm(sh, b + ".norm1", tr.c)
    _attn_shapes(sh, b + ".attn1", tr.c, tr.c)
    _norm(sh, b + ".norm2", tr.c)
    _attn_shapes(sh, b + ".attn2", tr.c, cross)
    _norm(sh, b + ".norm3", tr.c)
    _lin(sh, b + ".ff.net.0.proj", 8 * tr.c, tr.c)
    _lin(sh, b + ".ff.net.2", tr.c, 4 * tr.c)
    if tr.multiview:
        _norm(sh, b + ".norm4", tr.c)
        _attn_shapes(sh, b + ".attn4", tr.c, tr.c)
        _lin(sh, b + ".connector", tr.c, tr.c)
    _conv(sh, p + ".proj_out", tr.c, tr.c, 1)


def _encoder_shapes(sh, cfg, multiview):
    c0 = cfg.block_out_channels[0]
    temb = cfg.time_embed_dim
    _conv(sh, "conv_in", c0, cfg.in_channels, 3)
    _lin(sh, "time_embedding.linear_1", temb, c0)
    _lin(sh, "time_embedding.linear_2", temb, temb)
    for blk in down_blocks(cfg, multiview):
        for rs, tr in blk.layers:
            _resnet_shapes(sh, rs, temb)
            if tr is not None:
                _transformer_shapes(sh, tr, cfg.cross_attention_dim)
        if blk.sampler is not None:
            _conv(sh, blk.sampler.prefix, blk.sampler.c, blk.sampler.c, 3)
    r0, tr, r1 = mid_block(cfg, multiview)
    _resnet_shapes(sh, r0, temb)
    _transformer_shapes(sh, tr, cfg.cross_attention_dim)
    _resnet_shapes(sh, r1, temb)


def unet_param_shapes(cfg: UNetConfig) -> "OrderedDict[str, tuple]":
    sh = OrderedDict()
    _encoder_shapes(sh, cfg, cfg.multiview)
    temb = cfg.time_embed_dim
    for blk in up_blocks(cfg):
        for rs, tr in blk.layers:
            _resnet_shapes(sh, rs, temb)
            if tr is not None:
                _transformer_shapes(sh, tr, cfg.cross_attention_dim)
        if blk.sampler is not None:
            _conv(sh, blk.sampler.prefix, blk.sampler.c, blk.sampler.c, 3)
    _norm(sh, "conv_norm_out", cfg.block_out_channels[0])
    _conv(sh, "conv_out", cfg.out_channels, cfg.block_out_channels[0], 3)
    return sh


def map_encoder_layers(cfg: ControlNetConfig):
    """(name, cin, cout, stride(h,w), pad(h,w)) of BEVControlNetConditioningEmbedding (map_embedder.py:28-64) or, with
    cfg.map_embedding_size set, of BEVControlNetConditioningEmbeddingPlus (:79-126: all pads 1, first strided block stride 1,
    and an AdaptiveAvgPool2d(cfg.map_embedding_size) as `blocks.{last}` ahead of conv_out -- it has no parameters and is
    not listed here; engine / oracle insert it)."""
    ch = cfg.conditioning_embedding_out_channels
    plus = cfg.map_embedding_size is not None
    layers = [("controlnet_cond_embedding.conv_in", cfg.map_size[0], ch[0], (1, 1), (1, 1))]
    bi = 0
    for i in range(len(ch) - 2):
        layers.append((f"controlnet_cond_embedding.blocks.{bi}", ch[i], ch[i], (1, 1), (1, 1)))
        if plus:
            st = (1, 1) if i == 0 else (2, 2)
            layers.append((f"controlnet_cond_embedding.blocks.{bi + 1}", ch[i], ch[i + 1], st, (1, 1)))
        else:
            layers.append((f"controlnet_cond_embedding.blocks.{bi + 1}", ch[i], ch[i + 1], (2, 2), (2, 1)))
        bi += 2
    layers.append((f"controlnet_cond_embedding.blocks.{bi}", ch[-2], ch[-2], (1, 1), (1, 1) if plus else (2, 1)))
    layers.append((f"controlnet_cond_embedding.blocks.{bi + 1}", ch[-2], ch[-1], (2, 1), (1, 1) if plus else (2, 1)))
    layers.append(("controlnet_cond_embedding.conv_out", ch[-1], cfg.block_out_channels[0], (1, 1), (1, 1)))
    return layers


def controlnet_residual_channels(cfg) -> List[int]:
    """Channels of the 1 + sum(layers + sampler) skip tensors (unet_addon_rawbox.py:221-259)."""
    chans = [cfg.block_out_channels[0]]
    for i, _ in enumerate(cfg.down_block_types):
        c = cfg.block_out_channels[i]
        chans += [c] * cfg.layers_per_block
        if i != len(cfg.block_out_channels) - 1:
            chans.append(c)
    return chans


def controlnet_param_shapes(cfg: ControlNetConfig) -> "OrderedDict[str, tuple]":
    sh = OrderedDict()
    _lin(sh, "cam2token", cfg.camera_out_dim, cfg.camera_in_dim)
    sh["uncond_cam.weight"] = (1, cfg.uncond_cam_in_dim[0] * cfg.uncond_cam_in_dim[1])
    _encoder_shapes(sh, cfg, False)
    for name, ci, co, _, _ in map_encoder_layers(cfg):
        _conv(sh, name, co, ci, 3)
    fdim = 3 * (1 + 2 * cfg.bbox_num_freqs) * cfg.bbox_points
    pd = cfg.bbox_proj_dims
    _lin(sh, "bbox_embedder.bbox_proj", pd[0], fdim)
    _lin(sh, "bbox_embedder.second_linear.0", pd[1], pd[0] + cfg.bbox_class_token_dim)
    _lin(sh, "bbox_embedder.second_linear.2", pd[2], pd[1])
    _lin(sh, "bbox_embedder.second_linear.4", pd[3], pd[2])
    sh["bbox_embedder._class_tokens"] = (cfg.bbox_n_classes, cfg.bbox_class_token_dim)  # buffer
    sh["bbox_embedder.null_class_feature"] = (cfg.bbox_class_token_dim,)
    sh["bbox_embedder.null_pos_feature"] = (fdim,)
    for i, c in enumerate(controlnet_residual_channels(cfg)):
        _conv(sh, f"controlnet_down_blocks.{i}", c, c, 1)
    _conv(sh, "controlnet_mid_block", cfg.block_out_channels[-1], cfg.block_out_channels[-1], 1)
    return sh


# ------------------------------------------------------------------------------------------ VAE (SURVEY §8 f2, f7)
@dataclass
class VaeConfig:
    """AutoencoderKL config of SD-1.5 (third_party/diffusers/src/diffusers/models/autoencoder_kl.py:66-82): the decoder
    turns generated latents into views (pipeline_bev_controlnet.py:100-112), the encoder turns camera images into given-view
    latents (demo/run_cond_on_view.py:80-85)."""
    in_channels: int = 3
    out_channels: int = 3
    down_block_types: Tuple[str, ...] = ("DownEncoderBlock2D",) * 4
    up_block_types: Tuple[str, ...] = ("UpDecoderBlock2D",) * 4
    block_out_channels: Tuple[int, ...] = (128, 256, 512, 512)
    layers_per_block: int = 2
    act_fn: str = "silu"
    latent_channels: int = 4
    norm_num_groups: int = 32
    sample_size: int = 512
    scaling_factor: float = 0.18215


def vae_decoder_blocks(cfg: VaeConfig):
    """[(prefix, [(resnet prefix, cin, cout)], upsampler prefix or None)] of Decoder.up_blocks (vae.py:193-219)."""
    rev = list(reversed(cfg.block_out_channels))
    blocks, out_c = [], rev[0]
    for i in range(len(rev)):
        prev, out_c = out_c, rev[i]
        res = [(f"decoder.up_blocks.{i}.resnets.{j}", prev if j == 0 else out_c, out_c) for j in range(cfg.layers_per_block + 1)]
        up = None if i == len(rev) - 1 else f"decoder.up_blocks.{i}.upsamplers.0.conv"
        blocks.append((f"decoder.up_blocks.{i}", res, up))
    return blocks


def vae_encoder_blocks(cfg: VaeConfig):
    """[(prefix, [(resnet prefix, cin, cout)], downsampler prefix or None)] of Encoder.down_blocks (vae.py:65-85): every
    block but the last ends in Downsample2D(padding=0), a 3x3 stride-2 conv after padding the bottom / right edge by one."""
    ch = cfg.block_out_channels
    blocks = []
    for i, out_c in enumerate(ch):
        prev = ch[max(i - 1, 0)]
        res = [(f"encoder.down_blocks.{i}.resnets.{j}", prev if j == 0 else out_c, out_c) for j in range(cfg.layers_per_block)]
        down = None if i == len(ch) - 1 else f"encoder.down_blocks.{i}.downsamplers.0.conv"
        blocks.append((f"encoder.down_blocks.{i}", res, down))
    return blocks


def _vae_resnet_shapes(sh, p, ci, co):
    _norm(sh, p + ".norm1", ci)
    _conv(sh, p + ".conv1", co, ci, 3)
    _norm(sh, p + ".norm2", co)
    _conv(sh, p + ".conv2", co, co, 3)
    if ci != co:
        _conv(sh, p + ".conv_shortcut", co, ci, 1)


def _vae_mid_shapes(sh, half: str, c_mid: int):
    a = f"{half}.mid_block.attentions.0"
    _norm(sh, a + ".group_norm", c_mid)
    for n in ("to_q", "to_k", "to_v", "to_out.0"):
        _lin(sh, f"{a}.{n}", c_mid, c_mid)
    _vae_resnet_shapes(sh, f"{half}.mid_block.resnets.0", c_mid, c_mid)
    _vae_resnet_shapes(sh, f"{half}.mid_block.resnets.1", c_mid, c_mid)


def vae_encoder_param_shapes(cfg: VaeConfig) -> "OrderedDict[str, tuple]":
    """Encoder + quant_conv keys of AutoencoderKL.state_dict() (vae.py:39-106, autoencoder_kl.py:87-106): the encoder
    writes 2 x latent_channels moments (double_z)."""
    sh: "OrderedDict[str, tuple]" = OrderedDict()
    moments = 2 * cfg.latent_channels
    _conv(sh, "encoder.conv_in", cfg.block_out_channels[0], cfg.in_channels, 3)
    for _, resnets, down in vae_encoder_blocks(cfg):
        for p, ci, co in resnets:
            _vae_resnet_shapes(sh, p, ci, co)
        if down:
            _conv(sh, down, resnets[-1][2], resnets[-1][2], 3)
    _vae_mid_shapes(sh, "encoder", cfg.block_out_channels[-1])
    _norm(sh, "encoder.conv_norm_out", cfg.block_out_channels[-1])
    _conv(sh, "encoder.conv_out", moments, cfg.block_out_channels[-1], 3)
    _conv(sh, "quant_conv", moments, moments, 1)
    return sh


def vae_decoder_param_shapes(cfg: VaeConfig) -> "OrderedDict[str, tuple]":
    """Decoder + post_quant_conv keys of AutoencoderKL.state_dict() (vae.py:152-225, autoencoder_kl.py:107-108)."""
    sh: "OrderedDict[str, tuple]" = OrderedDict()
    c_mid = cfg.block_out_channels[-1]
    _conv(sh, "decoder.conv_in", c_mid, cfg.latent_channels, 3)
    for _, resnets, up in vae_decoder_blocks(cfg):
        for p, ci, co in resnets:
            _vae_resnet_shapes(sh, p, ci, co)
        if up:
            _conv(sh, up, resnets[-1][2], resnets[-1][2], 3)
    _vae_mid_shapes(sh, "decoder", c_mid)
    _norm(sh, "decoder.conv_norm_out", cfg.block_out_channels[0])
    _conv(sh, "decoder.conv_out", cfg.out_channels, cfg.block_out_channels[0], 3)
    _conv(sh, "post_quant_conv", cfg.latent_channels, cfg.latent_channels, 1)
    return sh


# ------------------------------------------------------------------------------------------ CLIP text encoder
@dataclass
class ClipTextConfig:
    """CLIPTextConfig of SD-1.5's text_encoder/config.json (CLIP ViT-L/14 text tower): pre-LN transformer with causal
    self-attention and a quick_gelu MLP (transformers models/clip/configuration_clip.py, modeling_clip.py)."""
    vocab_size: int = 49408
    hidden_size: int = 768
    intermediate_size: int = 3072
    num_hidden_layers: int = 12
    num_attention_heads: int = 12
    max_position_embeddings: int = 77
    hidden_act: str = "quick_gelu"
    layer_norm_eps: float = 1e-5
    bos_token_id: int = 0
    eos_token_id: int = 2
    pad_token_id: int = 1
    projection_dim: int = 768


def clip_text_param_shapes(cfg: ClipTextConfig) -> "OrderedDict[str, tuple]":
    """CLIPTextModel.state_dict() keys (196 at SD-1.5 size): text_model.embeddings.*, .encoder.layers.N.*, .final_layer_norm."""
    sh: "OrderedDict[str, tuple]" = OrderedDict()
    c, t = cfg.hidden_size, "text_model"
    sh[t + ".embeddings.token_embedding.weight"] = (cfg.vocab_size, c)
    sh[t + ".embeddings.position_embedding.weight"] = (cfg.max_position_embeddings, c)
    for i in range(cfg.num_hidden_layers):
        p = f"{t}.encoder.layers.{i}"
        for n in ("k_proj", "v_proj", "q_proj", "out_proj"):
            _lin(sh, f"{p}.self_attn.{n}", c, c)
        _norm(sh, p + ".layer_norm1", c)
        _lin(sh, p + ".mlp.fc1", cfg.intermediate_size, c)
        _lin(sh, p + ".mlp.fc2", c, cfg.intermediate_size)
        _norm(sh, p + ".layer_norm2", c)
    _norm(sh, t + ".final_layer_norm", c)
    return sh


BUFFER_KEYS = {"bbox_embedder._class_tokens"}


# ------------------------------------------------------------------------------------------ deterministic weights
def synthetic_state_dict(shapes, seed: int = 0, scale: float = 1.0):
    """Name-keyed deterministic weights (numpy Philox per tensor name) so that the reference model built in the
    oracle container and our model on the GPU box hold bit-identical fp32 parameters without shipping them.
    Every tensor is non-zero: the reference zero-initialises `connector`, the ControlNet 1x1 convs and the map
    encoder's conv_out (controlnet.py:585-588), which would hide cross-view / ControlNet bugs."""
    import zlib

    import numpy as np
    import torch

    def make(item):
        name, shape = item
        rng = np.random.Generator(np.random.Philox(key=(seed << 32) + zlib.crc32(name.encode())))
        if name.endswith(".weight") and len(shape) >= 2:
            fan_in = int(np.prod(shape[1:]))
            # the camera / box encoders see raw metric inputs (fx ~ 1.27e3 px, box corners +-50 m); a trained
            # checkpoint keeps their tokens O(1-10) like the CLIP tokens beside them, so do the synthetic weights
            # (otherwise one token saturates every conditioning softmax and bf16 parity becomes a coin flip)
            gain = {"cam2token.weight": 0.02, "bbox_embedder.bbox_proj.weight": 0.1}.get(name, 1.0)
            a = rng.standard_normal(shape, dtype=np.float32) * (gain * scale / np.sqrt(fan_in))
        elif name.endswith(".weight"):  # norm gains
            a = 1.0 + 0.1 * rng.standard_normal(shape, dtype=np.float32)
        elif "_class_tokens" in name:
            a = rng.standard_normal(shape, dtype=np.float32)
        else:  # biases, null features
            a = 0.05 * rng.standard_normal(shape, dtype=np.float32)
        return name, torch.from_numpy(np.ascontiguousarray(a.astype(np.float32)))

    # one independent Philox stream per tensor name: order- and thread-count-independent, so the tensors are generated
    # in parallel (numpy releases the GIL while filling)
    import os
    from concurrent.futures import ThreadPoolExecutor
    items = list(shapes.items())
    with ThreadPoolExecutor(max_workers=min(16, os.cpu_count() or 1)) as ex:
        sd = OrderedDict(ex.map(make, items))
    return sd


# ------------------------------------------------------------------------------------------ FID InceptionV3
# The FID variant of torchvision's Inception3 as magicdrive/misc/inception.py:197-221 (fid_inception_v3) assembles it:
# num_classes=1008, aux_logits=False, Mixed_5b-5d = FIDInceptionA, Mixed_6b-6e = FIDInceptionC, Mixed_7b / 7c =
# FIDInceptionE_1 / _2, Mixed_6a / 7a = torchvision's InceptionB / InceptionD.  Every BasicConv2d is a bias-free conv,
# BatchNorm2d(eps=0.001) and ReLU (torchvision models/inception.py BasicConv2d).
INCEPTION_BN_EPS = 1e-3
INCEPTION_SIZE = 299
INCEPTION_DIMS = (64, 192, 768, 2048)  # channels of the four output blocks (inception.py:24-29)


@dataclass(frozen=True)
class InceptionConv:
    name: str  # torchvision module name (the pytorch-fid weights file's keys), e.g. "Mixed_6b.branch7x7_2"
    cin: int
    cout: int
    kh: int
    kw: int
    stride: int = 1
    ph: int = 0
    pw: int = 0


# (module, kind, in_channels, pool_features / channels_7x7) of InceptionV3 blocks 2 and 3 (inception.py:103-124)
INCEPTION_MIXED = (
    ("Mixed_5b", "A", 192, 32), ("Mixed_5c", "A", 256, 64), ("Mixed_5d", "A", 288, 64), ("Mixed_6a", "B", 288, 0),
    ("Mixed_6b", "C", 768, 128), ("Mixed_6c", "C", 768, 160), ("Mixed_6d", "C", 768, 160), ("Mixed_6e", "C", 768, 192),
    ("Mixed_7a", "D", 768, 0), ("Mixed_7b", "E1", 1280, 0), ("Mixed_7c", "E2", 2048, 0),
)
# torchvision module names of each InceptionV3 block's layers (inception.py:84-124); pools carry no parameters
INCEPTION_BLOCKS = (
    ("Conv2d_1a_3x3", "Conv2d_2a_3x3", "Conv2d_2b_3x3"),
    ("Conv2d_3b_1x1", "Conv2d_4a_3x3"),
    ("Mixed_5b", "Mixed_5c", "Mixed_5d", "Mixed_6a", "Mixed_6b", "Mixed_6c", "Mixed_6d", "Mixed_6e"),
    ("Mixed_7a", "Mixed_7b", "Mixed_7c"),
)


def mixed_out_channels(kind: str, cin: int, arg: int) -> int:
    return {"A": 224 + arg, "B": 384 + 96 + cin, "C": 768, "D": 320 + 192 + cin, "E1": 2048, "E2": 2048}[kind]


def _mixed_convs(m: str, kind: str, cin: int, arg: int) -> List[InceptionConv]:
    """Convolutions of one Mixed block in torchvision's registration order (models/inception.py InceptionA-E)."""
    C = lambda s, ci, co, kh, kw, st=1, ph=0, pw=0: InceptionConv(f"{m}.{s}", ci, co, kh, kw, st, ph, pw)
    if kind == "A":
        return [C("branch1x1", cin, 64, 1, 1), C("branch5x5_1", cin, 48, 1, 1), C("branch5x5_2", 48, 64, 5, 5, 1, 2, 2),
                C("branch3x3dbl_1", cin, 64, 1, 1), C("branch3x3dbl_2", 64, 96, 3, 3, 1, 1, 1),
                C("branch3x3dbl_3", 96, 96, 3, 3, 1, 1, 1), C("branch_pool", cin, arg, 1, 1)]
    if kind == "B":
        return [C("branch3x3", cin, 384, 3, 3, 2), C("branch3x3dbl_1", cin, 64, 1, 1),
                C("branch3x3dbl_2", 64, 96, 3, 3, 1, 1, 1), C("branch3x3dbl_3", 96, 96, 3, 3, 2)]
    if kind == "C":
        c7 = arg
        return [C("branch1x1", cin, 192, 1, 1), C("branch7x7_1", cin, c7, 1, 1), C("branch7x7_2", c7, c7, 1, 7, 1, 0, 3),
                C("branch7x7_3", c7, 192, 7, 1, 1, 3, 0), C("branch7x7dbl_1", cin, c7, 1, 1),
                C("branch7x7dbl_2", c7, c7, 7, 1, 1, 3, 0), C("branch7x7dbl_3", c7, c7, 1, 7, 1, 0, 3),
                C("branch7x7dbl_4", c7, c7, 7, 1, 1, 3, 0), C("branch7x7dbl_5", c7, 192, 1, 7, 1, 0, 3),
                C("branch_pool", cin, 192, 1, 1)]
    if kind == "D":
        return [C("branch3x3_1", cin, 192, 1, 1), C("branch3x3_2", 192, 320, 3, 3, 2),
                C("branch7x7x3_1", cin, 192, 1, 1), C("branch7x7x3_2", 192, 192, 1, 7, 1, 0, 3),
                C("branch7x7x3_3", 192, 192, 7, 1, 1, 3, 0), C("branch7x7x3_4", 192, 192, 3, 3, 2)]
    return [C("branch1x1", cin, 320, 1, 1), C("branch3x3_1", cin, 384, 1, 1), C("branch3x3_2a", 384, 384, 1, 3, 1, 0, 1),
            C("branch3x3_2b", 384, 384, 3, 1, 1, 1, 0), C("branch3x3dbl_1", cin, 448, 1, 1),
            C("branch3x3dbl_2", 448, 384, 3, 3, 1, 1, 1), C("branch3x3dbl_3a", 384, 384, 1, 3, 1, 0, 1),
            C("branch3x3dbl_3b", 384, 384, 3, 1, 1, 1, 0), C("branch_pool", cin, 192, 1, 1)]


def inception_convs(last_block: int = 3) -> "OrderedDict[str, Tuple[str, InceptionConv]]":
    """torchvision name -> (InceptionV3 wrapper prefix `blocks.{i}.{j}[.branch]`, conv) for blocks 0..last_block."""
    stem = {"Conv2d_1a_3x3": InceptionConv("Conv2d_1a_3x3", 3, 32, 3, 3, 2),
            "Conv2d_2a_3x3": InceptionConv("Conv2d_2a_3x3", 32, 32, 3, 3),
            "Conv2d_2b_3x3": InceptionConv("Conv2d_2b_3x3", 32, 64, 3, 3, 1, 1, 1),
            "Conv2d_3b_1x1": InceptionConv("Conv2d_3b_1x1", 64, 80, 1, 1),
            "Conv2d_4a_3x3": InceptionConv("Conv2d_4a_3x3", 80, 192, 3, 3)}
    mixed = {m: (kind, cin, arg) for m, kind, cin, arg in INCEPTION_MIXED}
    out = OrderedDict()
    for i, mods in enumerate(INCEPTION_BLOCKS[: last_block + 1]):
        for j, m in enumerate(mods):
            if m in stem:
                out[m] = (f"blocks.{i}.{j}", stem[m])
            else:
                for cv in _mixed_convs(m, *mixed[m]):
                    out[cv.name] = (f"blocks.{i}.{j}.{cv.name.split('.', 1)[1]}", cv)
    return out


INCEPTION_BN_BUFFERS = ("running_mean", "running_var", "num_batches_tracked")


def inception_param_shapes(last_block: int = 3) -> "OrderedDict[str, tuple]":
    """State-dict keys and shapes of magicdrive/misc/inception.py InceptionV3 built with max(output_blocks) = last_block."""
    sh = OrderedDict()
    for prefix, cv in inception_convs(last_block).values():
        sh[prefix + ".conv.weight"] = (cv.cout, cv.cin, cv.kh, cv.kw)
        for s in ("weight", "bias", "running_mean", "running_var"):
            sh[f"{prefix}.bn.{s}"] = (cv.cout,)
        sh[prefix + ".bn.num_batches_tracked"] = ()
    return sh


def inception_synthetic_state_dict(last_block: int = 3, seed: int = 0):
    """Seeded weights under the wrapper's names (Philox per tensor name, like arch.synthetic_state_dict) with sane
    BatchNorm statistics: gains near 1, running_var in [0.5, 1.5], so the features are neither degenerate nor exploding."""
    import zlib

    import numpy as np
    import torch
    sd = OrderedDict()
    for name, shape in inception_param_shapes(last_block).items():
        rng = np.random.Generator(np.random.Philox(key=(seed << 32) + zlib.crc32(name.encode())))
        if name.endswith("num_batches_tracked"):
            sd[name] = torch.zeros((), dtype=torch.long)
            continue
        if name.endswith("conv.weight"):
            a = rng.standard_normal(shape, dtype=np.float32) * np.float32(np.sqrt(2.0 / np.prod(shape[1:])))
        elif name.endswith("bn.weight"):
            a = 1.0 + 0.1 * rng.standard_normal(shape, dtype=np.float32)
        elif name.endswith("running_var"):
            a = rng.uniform(0.5, 1.5, shape).astype(np.float32)
        else:  # bn.bias, running_mean
            a = 0.1 * rng.standard_normal(shape, dtype=np.float32)
        sd[name] = torch.from_numpy(np.ascontiguousarray(a.astype(np.float32)))
    return sd
