"""FID Inception on the sm_90a path: the convolution shapes, K tails, ReLU epilogue, pools and input kernel against float64
with guarded column-slice outputs, then the whole network against the fp32 oracle (oracle/fid_inception.py), graph replay,
the FID yardstick and FIDStatistics against the PNG route."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from magicdrive_b200 import arch, fid, ops  # noqa: E402
from magicdrive_b200.models import InceptionV3  # noqa: E402
from magicdrive_b200.params import pack_conv_weight_k64  # noqa: E402
from oracle import fid_inception as fid_oracle  # noqa: E402
from tests.common import record, rel_l2  # noqa: E402
from tests.test_kernel_edges_gpu import Guarded, _close  # noqa: E402

BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64


def _conv_case(*, n, h, w, c0, co, kh, kw, stride=1, ph=0, pw=0, relu=True, ld_in=None, ld_out=None, col0=0, seed=0, c1=0,
               **extra):
    """One guarded ReLU conv with K64-packed weights against float64; c1 > 0 adds a second A source (channel concat).
    Returns the max error relative to max |ref|."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    ld_in = ld_in or c0
    x = (torch.randn(n * h * w, ld_in, device="cuda", generator=g)).to(BF16)
    x1 = (torch.randn(n * h * w, c1 + 8, device="cuda", generator=g)).to(BF16) if c1 else None
    cin = c0 + c1
    wt = (torch.randn(co, cin, kh, kw, device="cuda", generator=g) / math.sqrt(cin * kh * kw)).to(BF16).float()
    b = torch.randn(co, device="cuda", generator=g) * 0.5
    ho, wo = (h + 2 * ph - kh) // stride + 1, (w + 2 * pw - kw) // stride + 1
    out = Guarded(n * ho * wo, co, BF16, ld=ld_out or co, col0=col0)
    ops.gemm_conv(x, pack_conv_weight_k64(wt, [c0, c1] if c1 else None), n_img=n, h_in=h, w_in=w, c0=c0, lda0=ld_in,
                  a1=x1, c1=c1, lda1=c1 + 8 if c1 else 0, n_out=co, taps_h=kh, taps_w=kw, stride=stride, pad_h=ph, pad_w=pw,
                  bias=b, relu=relu, out=out.out, ldo=out.ld, **extra)
    xi = x[:, :c0].to(F64)
    if c1:
        xi = torch.cat([xi, x1[:, :c1].to(F64)], 1)
    xi = xi.view(n, h, w, cin).permute(0, 3, 1, 2)
    ref = F.conv2d(xi, wt.to(F64), b.to(F64), stride=stride, padding=(ph, pw)).permute(0, 2, 3, 1).reshape(-1, co)
    if relu:
        assert (ref < 0).any(), "the case must have negative pre-activations"
        ref = ref.clamp_min(0)
    out.check(f"conv {kh}x{kw}")
    _close(out.out, ref, f"conv {kh}x{kw} s{stride} c0={c0} c1={c1}")
    return ((out.out.to(F64) - ref).abs().max() / ref.abs().max()).item()


# (n, h, w, c0, co, kh, kw, stride, ph, pw): every kind of Inception convolution at its real shape
INCEPTION_CONVS = {
    "1a_3x3_s2_299": (2, 299, 299, 8, 32, 3, 3, 2, 0, 0),
    "2a_3x3_valid": (2, 149, 149, 32, 32, 3, 3, 1, 0, 0),
    "3b_1x1_c80": (2, 73, 73, 64, 80, 1, 1, 1, 0, 0),
    "4a_3x3_c80": (2, 73, 73, 80, 192, 3, 3, 1, 0, 0),
    "5x5_c48": (3, 35, 35, 48, 64, 5, 5, 1, 2, 2),
    "6a_3x3_s2_35": (3, 35, 35, 288, 384, 3, 3, 2, 0, 0),
    "1x7_c160": (3, 17, 17, 160, 160, 1, 7, 1, 0, 3),
    "7x1_c160": (3, 17, 17, 160, 192, 7, 1, 1, 3, 0),
    "7a_3x3_s2_17": (3, 17, 17, 192, 320, 3, 3, 2, 0, 0),
    "1x3_c384": (3, 8, 8, 384, 384, 1, 3, 1, 0, 1),
    "3x1_c384": (3, 8, 8, 384, 384, 3, 1, 1, 1, 0),
    "3x3_c448": (3, 8, 8, 448, 384, 3, 3, 1, 1, 1),
}


@pytest.mark.parametrize("case", list(INCEPTION_CONVS))
def test_inception_conv_kinds(cuda_lib, case):
    n, h, w, c0, co, kh, kw, s, ph, pw = INCEPTION_CONVS[case]
    # written into a column slice of a wider buffer, as the Mixed blocks do
    e = _conv_case(n=n, h=h, w=w, c0=c0, co=co, kh=kh, kw=kw, stride=s, ph=ph, pw=pw, ld_out=co + 64, col0=32)
    record(f"[parity] fid conv {case}: max err / max |ref| {e:.3e}")


@pytest.mark.parametrize("c0", [8, 32, 48, 80, 96, 160, 288, 448])
@pytest.mark.parametrize("taps", [1, 3])
def test_k_tails(cuda_lib, c0, taps):
    # input read from a column slice (lda > c0): the channels past c0 are real data the TMA must not read
    e = _conv_case(n=2, h=19, w=23, c0=c0, co=96, kh=taps, kw=taps, ph=taps // 2, pw=taps // 2, ld_in=c0 + 16)
    record(f"[parity] fid K tail c0={c0} taps={taps}: max err / max |ref| {e:.3e}")


@pytest.mark.parametrize("c0,c1", [(80, 48), (160, 96), (64, 40)])
@pytest.mark.parametrize("taps", [1, 3])
def test_k_tails_two_sources(cuda_lib, c0, c1, taps):
    """Partial K blocks on both A sources: weights packed per source at 64-multiples (pack_conv_weight_k64 splits)."""
    e = _conv_case(n=2, h=13, w=21, c0=c0, c1=c1, co=64, kh=taps, kw=taps, ph=taps // 2, pw=taps // 2, ld_in=c0 + 8)
    record(f"[parity] fid K tail two sources c0={c0} c1={c1} taps={taps}: max err / max |ref| {e:.3e}")


@pytest.mark.parametrize("block_n", [64, 128, 160, 256])
@pytest.mark.parametrize("splits", [1, 3])
def test_relu_split_k(cuda_lib, block_n, splits):
    """ReLU through the split-K finalize pass and every tile width; the output has negative pre-activations."""
    e = _conv_case(n=1, h=8, w=8, c0=448, co=256, kh=3, kw=3, ph=1, pw=1, force_block_n=block_n, force_splits=splits)
    record(f"[parity] fid ReLU block_n={block_n} splits={splits}: max err / max |ref| {e:.3e}")


@pytest.mark.parametrize("mode,k,s,p", [(ops.POOL_MAX, 3, 2, 0), (ops.POOL_MAX, 3, 1, 1), (ops.POOL_AVG, 3, 1, 1),
                                        (ops.POOL_GLOBAL_AVG, 0, 0, 0)], ids=["max_s2", "max_s1p1", "avg_s1p1", "global"])
@pytest.mark.parametrize("shape", [(2, 147, 147, 64), (3, 17, 17, 768), (2, 8, 8, 2048), (1, 35, 35, 288)])
def test_pools(cuda_lib, mode, k, s, p, shape):
    n, h, w, c = shape
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn(n * h * w, c + 24, device="cuda", generator=g).to(BF16)
    xi = x[:, :c].to(F64).view(n, h, w, c).permute(0, 3, 1, 2)
    if mode == ops.POOL_GLOBAL_AVG:
        out = Guarded(n, c, F32, ld=c + 16, col0=8)
        ops.pool2d(x, n=n, h=h, w=w, c=c, ldx=c + 24, mode=mode, out=out.out, ldo=out.ld)
        ref = xi.mean((2, 3))
    else:
        ref = (F.max_pool2d(xi, k, s, p) if mode == ops.POOL_MAX else
               F.avg_pool2d(xi, k, s, p, count_include_pad=False))
        ho, wo = ref.shape[2:]
        ref = ref.permute(0, 2, 3, 1).reshape(-1, c)
        out = Guarded(n * ho * wo, c, BF16, ld=c + 40, col0=16)
        ops.pool2d(x, n=n, h=h, w=w, c=c, ldx=c + 24, mode=mode, k=k, stride=s, pad=p, out=out.out, ldo=out.ld)
    out.check("pool")
    e = ((out.out.to(F64) - ref).abs().max() / ref.abs().max()).item()
    record(f"[parity] fid pool mode={mode} k={k} s={s} p={p} {shape}: max err / max |ref| {e:.3e}")
    if mode == ops.POOL_MAX:
        assert torch.equal(out.out.to(F64), ref), "max pool must be exact"
    else:
        _close(out.out, ref, "pool")


@pytest.mark.parametrize("layout", ["nchw_f32", "nhwc_f32", "nhwc_bf16"])
@pytest.mark.parametrize("resize", [True, False])
@pytest.mark.parametrize("normalize", [True, False])
@pytest.mark.parametrize("quantize", [True, False])
def test_input_kernel(cuda_lib, layout, resize, normalize, quantize):
    g = torch.Generator(device="cuda").manual_seed(2)
    n, h, w = 3, 224, 400
    img = torch.rand(n, 3, h, w, device="cuda", generator=g)
    dt = BF16 if layout.endswith("bf16") else F32
    img = img.to(dt).float()
    src = (img.permute(0, 2, 3, 1) if layout.startswith("nhwc") else img).contiguous().to(dt)
    out = ops.fid_input(src, nhwc=layout.startswith("nhwc"), quantize=quantize, normalize=normalize,
                        size=(299, 299) if resize else None)
    if not resize:
        # Without resampling the output is the bf16 rounding of q = rint(255 x) / 255 (then 2q - 1): within half a bf16
        # step of the float64 value plus 1e-7 (one fp32 rounding of q).  A missing 8-bit rounding is off by up to 1/510,
        # beyond that bound wherever |q| < 1/2; without normalize the output must be bf16(q) bit for bit.
        # 255 x in fp32, as numpy_to_pil multiplies the fp32 images, then rint and an exact division
        q = torch.round(img * 255).clamp(0, 255).double() / 255 if quantize else img.double()
        q = 2 * q - 1 if normalize else q
        o = out.view(n, h, w, 8)
        assert torch.all(o[..., 3:] == 0)
        o = o[..., :3].permute(0, 3, 1, 2).double()
        half_step = torch.exp2(torch.floor(torch.log2(q.abs().clamp_min(2.0 ** -100))) - 8)
        err = (o - q).abs()
        assert torch.all(err <= half_step + 1e-7), (err - half_step).max().item()
        if not normalize:
            assert torch.equal(o.float().to(BF16), q.float().to(BF16)), "8-bit rounding not exact"
        record(f"[parity] fid input {layout} quantize={quantize} normalize={normalize} no resize: max err {err.max().item():.3e}")
        return
    ref = img.double()
    if quantize:
        ref = torch.round(ref.float() * 255).clamp(0, 255).double() / 255
    if resize:
        ref = F.interpolate(ref, size=(299, 299), mode="bilinear", align_corners=False)
    if normalize:
        ref = 2 * ref - 1
    ho, wo = ref.shape[2:]
    o = out.view(n, ho, wo, 8)
    assert torch.all(o[..., 3:] == 0)
    err = (o[..., :3].permute(0, 3, 1, 2).double() - ref).abs()
    record(f"[parity] fid input {layout} quantize={quantize} normalize={normalize} resize 299: max err {err.max().item():.3e}")
    assert err.max().item() <= 2.0 ** -8 * ref.abs().max().item() + 1e-6, err.max().item()


# ---------------------------------------------------------------------------------------------------- whole network
_SD = {}


def _model(blocks=(0, 1, 2, 3)):
    key = tuple(blocks)
    if key not in _SD:
        sd = arch.inception_synthetic_state_dict(max(blocks), seed=3)
        m = InceptionV3(list(blocks)).cuda()
        m.load_state_dict(sd)
        _SD[key] = (m, {k: v.cuda() for k, v in sd.items()})
    return _SD[key]


def _oracle(sd, x, blocks, dtype=F32, bs=25):
    with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):  # the fp32 oracle is fp32, not TF32
        outs = [fid_oracle.forward(sd, x[i:i + bs], blocks, dtype=dtype) for i in range(0, x.shape[0], bs)]
    return [torch.cat([o[j] for o in outs]) for j in range(len(blocks))]


@pytest.mark.parametrize("size", [(299, 299), (224, 400), (97, 131)])
@pytest.mark.parametrize("batch", [1, 6, 50])
def test_network_against_oracle(cuda_lib, size, batch):
    blocks = (0, 1, 2, 3)
    model, sd = _model(blocks)
    x = fid_oracle.images(batch, *size, seed=batch).cuda()
    ours = model(x)
    with torch.no_grad():
        ref = _oracle(sd, x, blocks)
        ref16 = _oracle(sd, x, blocks, dtype=BF16)
    for i, (o, r, r16) in enumerate(zip(ours, ref, ref16)):
        assert o.shape == r.shape and o.dtype == F32
        e, e16 = rel_l2(o, r), rel_l2(r16, r)
        record(f"[parity] fid inception {size[0]}x{size[1]} batch {batch} block {i}: err {e:.3e} vs bf16 oracle {e16:.3e}")
        assert e <= 1.0 * e16 + 5e-4, (i, e, e16)
    assert (ref[3] > 0).float().mean() > 0.2  # features are not dead
    if batch > 1:
        assert ref[3].std(0).mean() > 0  # and vary across images


def test_graph_replay_bitwise(cuda_lib):
    model, _ = _model()
    x = fid_oracle.images(6, 224, 400, seed=11).cuda()
    graphed = model(x)
    model.use_cuda_graph = False
    try:
        eager = model(x)
    finally:
        model.use_cuda_graph = True
    for a, b in zip(graphed, eager):
        assert torch.equal(a, b)
    record("[parity] fid inception graph replay vs eager: bitwise equal at every block")


def _fixture_err(out, entry, i):
    """rel-L2 of block i of `out` (NCHW) against the fixture: the features, or the per-channel means and sampled elements."""
    if i == 3:
        return rel_l2(out[:, :, 0, 0], entry["features"])
    o = out.cpu()
    return max(rel_l2(o.mean((2, 3)), entry[f"block{i}_mean"]),
               rel_l2(o.reshape(-1)[entry[f"block{i}_idx"]], entry[f"block{i}_val"]))


def test_network_against_reference_fixture(cuda_lib):
    """The reference's own InceptionV3 run (tests/golden/fid_inception.pt) at every block: ours within the bf16 yardstick."""
    from tests.common import golden
    fx = golden("fid_inception.pt")
    sd = arch.inception_synthetic_state_dict(3, fx["seed_weights"])
    model = InceptionV3([0, 1, 2, 3]).cuda()
    model.load_state_dict(sd)
    sdc = {k: v.cuda() for k, v in sd.items()}
    for key, img in fx["inputs"].items():
        x = img.float().cuda() / 255
        ours = model(x)
        with torch.no_grad():
            r16 = _oracle(sdc, x, (0, 1, 2, 3), dtype=BF16)
        for i in range(4):
            e, e16 = _fixture_err(ours[i], fx["taps"][key], i), _fixture_err(r16[i], fx["taps"][key], i)
            record(f"[parity] fid inception vs reference fixture {key} block {i}: err {e:.3e} vs bf16 oracle {e16:.3e}")
            assert e <= 1.0 * e16 + 5e-4, (key, i, e, e16)


def _perturbed(x, seed):
    g = torch.Generator().manual_seed(seed)
    noise = F.interpolate(torch.randn(x.shape[0], 3, 8, 8, generator=g), size=x.shape[2:], mode="bilinear")
    return ((x + 0.08 * noise).clamp(0, 1) * 255).round() / 255


@pytest.mark.parametrize("dims", [192, 2048])
def test_fid_yardstick(cuda_lib, dims):
    blk = InceptionV3.BLOCK_INDEX_BY_DIM[dims]
    model, sd = _model()
    a = fid_oracle.images(512, 128, 160, seed=21)
    b = _perturbed(a, 5)
    feats = {"ours": [], "fp32": [], "bf16": []}
    for xs in (a, b):
        fo, f32, f16 = [], [], []
        for i in range(0, 512, 64):
            x = xs[i:i + 64].cuda()
            fo.append(fid._to_features(model(x)[blk]))
            with torch.no_grad():
                f32.append(fid._to_features(_oracle(sd, x, (blk,), bs=64)[0]))
                f16.append(fid._to_features(_oracle(sd, x, (blk,), dtype=BF16, bs=64)[0]))
        for k, v in zip(("ours", "fp32", "bf16"), (fo, f32, f16)):
            feats[k].append(np.concatenate(v))
    val = {}
    for k, (fa, fb) in feats.items():
        val[k] = fid.calculate_frechet_distance(fa.mean(0), np.cov(fa, rowvar=False), fb.mean(0), np.cov(fb, rowvar=False))
    record(f"[parity] fid dims {dims}: ours {val['ours']:.5f} fp32 {val['fp32']:.5f} bf16 {val['bf16']:.5f}")
    assert abs(val["ours"] - val["fp32"]) <= abs(val["bf16"] - val["fp32"]) + 0.01 * val["fp32"]


def test_fid_statistics_matches_png_route(cuda_lib, tmp_path):
    """FIDStatistics on the denoiser's (S, n_cam, H, W, 3) device images == saving them as PNGs and get_activations."""
    from PIL import Image
    model, _ = _model((3,))  # get_activations reads the model's first output, as the reference's does
    g = torch.Generator(device="cuda").manual_seed(4)
    views = torch.rand(2, 6, 224, 400, 3, device="cuda", generator=g)
    st = fid.FIDStatistics(model, dims=2048)
    st.update(views)
    files = []
    for i, v in enumerate(views.reshape(-1, 224, 400, 3).cpu().numpy()):  # diffusers numpy_to_pil
        p = tmp_path / f"{i:02d}.png"
        Image.fromarray((v * 255).round().astype("uint8")).save(p)
        files.append(p)
    act = fid.get_activations(files, model, batch_size=12, dims=2048, device="cuda", num_workers=0)
    err = np.abs(st.activations() - act).max()
    record(f"[parity] FIDStatistics vs PNG route: max abs diff {err:.3e}")
    assert err <= 1e-6 * np.abs(act).max()
    mu, sigma = st.statistics()
    assert np.allclose(mu, act.mean(0)) and np.allclose(sigma, np.cov(act, rowvar=False))
