"""TEST INFRASTRUCTURE ONLY — a plain-torch fp32 restatement of the FID InceptionV3 (magicdrive/misc/inception.py:129-163
forward, :224-341 FIDInceptionA/C/E_1/E_2; torchvision models/inception.py BasicConv2d, InceptionB, InceptionD, Inception3
layer order), run from a state dict under the wrapper's names (`blocks.{i}.{j}...`).  It checks our kernels on the GPU (in
fp32, or in bf16 as the yardstick of what bf16 storage costs) and the engine's host logic on the CPU.  It walks the layer
table of magicdrive_b200/arch.py like the product does; tests/golden/fid_inception.pt, made by the reference's own
InceptionV3 (oracle/make_golden_fid.py), pins that table: tests/test_fid_cpu.py checks this restatement against it.
Kept in its own file next to oracle/clip_text.py; oracle/torch_oracle.py is unchanged."""
import torch
import torch.nn.functional as F

from magicdrive_b200 import arch


def _basic(sd, prefix, x, cv):
    """BasicConv2d: conv (no bias) -> BatchNorm2d(eps=0.001, eval) -> ReLU."""
    dt = x.dtype
    y = F.conv2d(x, sd[prefix + ".conv.weight"].to(dt), stride=cv.stride, padding=(cv.ph, cv.pw))
    y = F.batch_norm(y, sd[prefix + ".bn.running_mean"].to(dt), sd[prefix + ".bn.running_var"].to(dt),
                     sd[prefix + ".bn.weight"].to(dt), sd[prefix + ".bn.bias"].to(dt), False, 0.0, arch.INCEPTION_BN_EPS)
    return F.relu(y)


def forward(sd, inp, output_blocks=(3,), resize=True, normalize=True, dtype=torch.float32):
    """inp (N, 3, H, W) in [0, 1] -> list of the selected blocks' outputs (NCHW), as InceptionV3.forward."""
    last = max(output_blocks)
    convs = arch.inception_convs(last)
    c = lambda name, x: _basic(sd, convs[name][0], x, convs[name][1])
    x = inp.float()
    if resize:
        x = F.interpolate(x, size=(299, 299), mode="bilinear", align_corners=False)
    if normalize:
        x = 2 * x - 1
    x = x.to(dtype)
    avg = lambda t: F.avg_pool2d(t, 3, stride=1, padding=1, count_include_pad=False)
    outs = []
    for i in range(last + 1):
        if i < 2:
            for m in arch.INCEPTION_BLOCKS[i]:
                x = c(m, x)
            x = F.max_pool2d(x, 3, stride=2)
        for m, kind, _, _ in (arch.INCEPTION_MIXED[:8] if i == 2 else arch.INCEPTION_MIXED[8:] if i == 3 else ()):
            if kind == "A":
                br = [c(m + ".branch1x1", x), c(m + ".branch5x5_2", c(m + ".branch5x5_1", x)),
                      c(m + ".branch3x3dbl_3", c(m + ".branch3x3dbl_2", c(m + ".branch3x3dbl_1", x))),
                      c(m + ".branch_pool", avg(x))]
            elif kind == "B":
                br = [c(m + ".branch3x3", x),
                      c(m + ".branch3x3dbl_3", c(m + ".branch3x3dbl_2", c(m + ".branch3x3dbl_1", x))),
                      F.max_pool2d(x, 3, stride=2)]
            elif kind == "C":
                t = c(m + ".branch7x7dbl_1", x)
                for j in (2, 3, 4, 5):
                    t = c(f"{m}.branch7x7dbl_{j}", t)
                br = [c(m + ".branch1x1", x), c(m + ".branch7x7_3", c(m + ".branch7x7_2", c(m + ".branch7x7_1", x))), t,
                      c(m + ".branch_pool", avg(x))]
            elif kind == "D":
                t = c(m + ".branch7x7x3_3", c(m + ".branch7x7x3_2", c(m + ".branch7x7x3_1", x)))
                br = [c(m + ".branch3x3_2", c(m + ".branch3x3_1", x)), c(m + ".branch7x7x3_4", t),
                      F.max_pool2d(x, 3, stride=2)]
            else:
                t = c(m + ".branch3x3_1", x)
                t2 = c(m + ".branch3x3dbl_2", c(m + ".branch3x3dbl_1", x))
                pool = avg(x) if kind == "E1" else F.max_pool2d(x, 3, stride=1, padding=1)
                br = [c(m + ".branch1x1", x), c(m + ".branch3x3_2a", t), c(m + ".branch3x3_2b", t),
                      c(m + ".branch3x3dbl_3a", t2), c(m + ".branch3x3dbl_3b", t2), c(m + ".branch_pool", pool)]
            x = torch.cat(br, 1)
        if i == 3:
            x = F.adaptive_avg_pool2d(x, (1, 1))
        if i in output_blocks:
            outs.append(x.float())
    return outs


def images(n, h, w, seed=0):
    """Procedural [0, 1] images (n, 3, h, w): smooth gradients and blobs plus noise, stored at 8-bit levels."""
    g = torch.Generator().manual_seed(seed)
    yy, xx = torch.meshgrid(torch.linspace(0, 1, h), torch.linspace(0, 1, w), indexing="ij")
    out = []
    for _ in range(n):
        f = torch.rand(3, 4, generator=g) * 6
        base = torch.stack([0.5 + 0.5 * torch.sin(f[c, 0] * xx + f[c, 1] * yy + f[c, 2]) for c in range(3)])
        img = 0.7 * base + 0.3 * torch.rand(3, h, w, generator=g)
        out.append(img)
    return (torch.stack(out) * 255).round() / 255
