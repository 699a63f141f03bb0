"""Map images and mosaics on the sm_90a path: visualize_maps, concat_views and camera_views_u8 against the reference's own
images (tests/golden/map_visualizer.pt) and against the restatement (oracle/map_visualizer.py) on seeded batches, byte
for byte, and save_run_images' files against Pillow's."""
import os

import numpy as np
import pytest
import torch
from PIL import Image

pytestmark = pytest.mark.gpu

from magicdrive_b200 import box_overlay, ops, visualize  # noqa: E402
from oracle import fid_protocol, map_visualizer as O  # noqa: E402
from oracle.make_golden_box_overlay import backgrounds, load as load_boxes  # noqa: E402
from oracle.make_golden_map_visualizer import fake_legend, load, sha  # noqa: E402
from tests.common import GOLDEN  # noqa: E402
from tests.test_box_overlay_cpu import expected  # noqa: E402
from tests.test_visualize_cpu import ERRORS  # noqa: E402

FX = load(os.path.join(GOLDEN, "map_visualizer.pt"))


def _recording(calls):
    def legend(names, size):
        calls.append((names, size))
        return fake_legend(names, size)
    return legend


def test_reference_fixture_byte_for_byte(cuda_lib):
    """Every fixture case, batched by map shape and target size, in fp32 and uint8."""
    groups = {}
    for c in FX["maps"]:
        groups.setdefault((c["map"].shape, c["target_size"]), []).append(c)
    for (shape, target), cases in groups.items():
        for dtype in (torch.float32, torch.uint8):
            maps = torch.from_numpy(np.stack([c["map"] for c in cases])).to("cuda", dtype)
            calls = []
            got = visualize.visualize_maps(maps, FX["map_classes"], FX["object_classes"], target, _recording(calls))
            for c, img in zip(cases, got):
                a = img.cpu().numpy()
                assert a.shape == tuple(c["out_shape"]) and sha(a) == c["sha256"], c["name"]
                if "out" in c:
                    assert np.array_equal(a, c["out"]), c["name"]
            # each distinct set the reference passed to its legend, drawn at most once per process
            assert {n for n, _ in calls} <= {frozenset(c["legend_names"]) for c in cases}
            assert len(calls) == len(set(calls))


@pytest.mark.parametrize("B,side,C,target,dtype", [
    (1, 200, 18, 400, torch.float32), (3, 97, 18, 300, torch.uint8), (16, 97, 8, 150, torch.bool),
    (5, 200, 26, 800, torch.float32), (2, 97, 26, 150, torch.float32), (7, 400, 18, 400, torch.uint8),
    (4, 64, 18, 300, torch.bool), (9, 200, 8, 300, torch.float32)])
def test_seeded_batches_equal_oracle(cuda_lib, B, side, C, target, dtype):
    """Seeded maps, some without any dynamic layer set, with non-binary aux layers past the dynamic ones."""
    rng = np.random.default_rng([B, side, C, target])
    maps = (rng.random((B, C, side, side)) < rng.uniform(0.02, 0.4, (B, C, 1, 1))).astype(np.float32)
    maps[::3, 8:18] = 0
    if C > 18:
        maps[:, 18:] = rng.normal(size=(B, C - 18, side, side))  # ignored, as the reference's slices ignore them
    x = torch.from_numpy(maps)
    if dtype != torch.float32:
        x = torch.where(torch.arange(C).view(1, C, 1, 1) < 18, x, 0).to(dtype)
    n0 = ops.launch_count()
    got = visualize.visualize_maps(x.cuda(), target_size=target, legend=fake_legend)
    assert ops.launch_count() - n0 == (2 if visualize.resized_side(side, target) == side else 4)
    for b in range(B):
        want, _ = O.visualize_map(x[b].to(torch.float32).numpy()[:18], visualize.NUSCENES_MAP_CLASSES,
                                  visualize.NUSCENES_OBJECT_CLASSES, target, fake_legend)
        assert np.array_equal(got[b].cpu().numpy(), want), b


def test_errors_on_the_device(cuda_lib):
    m = torch.zeros(3, 18, 50, 50, device="cuda")
    m[2, 4, 10, 10] = 0.5
    with pytest.raises(ValueError, match="map 2 holds values other than 0 and 1"):
        visualize.visualize_maps(m, legend=fake_legend)
    m[2, 4, 10, 10] = 1
    with pytest.raises(ValueError, match="'lane' is not in list"):
        visualize.visualize_maps(m, list(visualize.NUSCENES_MAP_CLASSES[:4]) + ["lane"] + ["walkway"] * 3,
                                 legend=fake_legend)
    with pytest.raises(KeyError, match="divider"):
        visualize.visualize_maps(m, ["drivable_area"] * 4 + ["divider"] + ["walkway"] * 3, legend=fake_legend)
    with pytest.raises(ValueError, match="does not fit"):
        visualize.visualize_maps(torch.zeros(1, 18, 97, 97, device="cuda"), target_size=400, legend=fake_legend)


@pytest.mark.parametrize("name", sorted(ERRORS))
@pytest.mark.parametrize("dtype", [torch.float32, torch.uint8])
def test_error_cases_on_the_device(cuda_lib, name, dtype):
    """The reference's first error on each case (tests/test_visualize_cpu.py holds the cases to the reference), among
    them a colourless static class drawn only under an object."""
    m, classes, objs, exc, msg = ERRORS[name]
    with pytest.raises(exc, match=msg):
        visualize.visualize_maps(m.to("cuda", dtype), classes, objs, 48, legend=fake_legend)


@pytest.mark.parametrize("dtype,bad", [(torch.float32, 2.0), (torch.float32, -1.0), (torch.float32, float("nan")),
                                       (torch.float32, float("inf")), (torch.float32, 1e-40), (torch.float32, -1e-45),
                                       (torch.uint8, 2), (torch.uint8, 255)])
@pytest.mark.parametrize("channel", [3, 12])
def test_non_binary_values_on_the_device(cuda_lib, dtype, bad, channel):
    """Values tested on their bits: denormals are not 0 in the kernel's flush-to-zero build.  Past the dynamic layers a
    value is never read."""
    m = torch.zeros(2, 26, 40, 40, dtype=dtype)
    m[:, 0, :20] = 1
    m[1, channel, 7, 9] = bad
    with pytest.raises(ValueError, match="map 1 holds values other than 0 and 1"):
        visualize.visualize_maps(m.cuda(), target_size=80, legend=fake_legend)
    m[1, channel, 7, 9] = 0
    m[1, 21, 7, 9] = bad
    got = visualize.visualize_maps(m.cuda(), target_size=80, legend=fake_legend)
    want, _ = O.visualize_map(m[1, :18].to(torch.float32).numpy(), visualize.NUSCENES_MAP_CLASSES,
                              visualize.NUSCENES_OBJECT_CLASSES, 80, fake_legend)
    assert np.array_equal(got[1].cpu().numpy(), want)


def test_negative_zero_is_an_unset_layer(cuda_lib):
    m = (torch.rand(2, 18, 40, 40, generator=torch.Generator().manual_seed(5)) < 0.2).float()
    z = torch.where(m == 0, torch.tensor(-0.0), m)
    a = visualize.visualize_maps(m.cuda(), target_size=80, legend=fake_legend)
    b = visualize.visualize_maps(z.cuda(), target_size=80, legend=fake_legend)
    assert all(torch.equal(x, y) for x, y in zip(a, b))


def test_mosaics_equal_reference_fixture(cuda_lib):
    for c in FX["mosaics"]:
        got = visualize.concat_views(torch.from_numpy(c["views"]).cuda()[None].expand(2, -1, -1, -1, -1), c["oneline"])
        assert np.array_equal(got[1].cpu().numpy(), c["out"]), (c["V"], c["C"], c["oneline"])


@pytest.mark.parametrize("V,H,W,C", [(5, 31, 57, 3), (6, 224, 400, 4), (7, 9, 13, 4), (2, 16, 16, 3), (9, 17, 5, 3)])
@pytest.mark.parametrize("oneline", [False, True])
def test_mosaics_equal_oracle(cuda_lib, V, H, W, C, oneline):
    if V < 5 and not oneline:
        pytest.skip("the reference has no two-row mosaic of fewer than 5 views")
    rng = np.random.default_rng([V, H, W, C])
    views = rng.integers(0, 256, (3, V, H, W, C), dtype=np.uint8)
    got = visualize.concat_views(torch.from_numpy(views).cuda(), oneline).cpu().numpy()
    assert np.array_equal(got, np.stack([O.concat_6_views(v, oneline) for v in views]))
    if C == 3:  # fp32 [0, 1] views, as decode_latents returns them, rounded as numpy_to_pil does
        f = rng.random((3, V, H, W, 3), dtype=np.float32)
        got = visualize.concat_views(torch.from_numpy(f).cuda(), oneline).cpu().numpy()
        assert np.array_equal(got, np.stack([O.concat_6_views(fid_protocol.to_u8(v), oneline) for v in f]))


def test_camera_views_equal_reference_fixture_and_oracle(cuda_lib):
    m = FX["m11"]
    x = m["x"][None, None].expand(2, 6, -1, -1, -1).contiguous()
    got = visualize.camera_views_u8(x.cuda()).cpu()
    assert bool((got == m["out"]).all())
    rng = np.random.default_rng(7)
    x = rng.uniform(-1, 1, (2, 6, 3, 224, 400)).astype(np.float32)
    got = visualize.camera_views_u8(torch.from_numpy(x).cuda()).cpu().numpy()
    assert np.array_equal(got, O.m11_to_u8(x))


def test_box_mosaics_equal_reference(cuda_lib):
    """The `_ori_box` / `_gen{t}_box` mosaics of the transparent box layers, against the reference's own layers."""
    fx = load_boxes(os.path.join(GOLDEN, "box_overlay.pt"))
    cases = fx["cases"]
    bg = backgrounds(len(cases), fx["seed"])
    layers = box_overlay.show_box_on_views(torch.from_numpy(bg).cuda(), cases, fx["classes"], transparent_bg=True)
    got = visualize.concat_views(layers).cpu().numpy()
    for s, (c, b) in enumerate(zip(cases, bg)):
        assert np.array_equal(got[s], O.concat_6_views(expected(c, b, True))), s


def test_save_run_images_files_equal_pillow(cuda_lib, tmp_path):
    rng = np.random.default_rng(11)
    demo = [c["map"] for c in FX["maps"] if c["name"] in ("demo0@400", "demo3@400")]
    maps = visualize.visualize_maps(torch.from_numpy(np.stack(demo)).cuda(), legend=fake_legend)
    px = torch.from_numpy(rng.uniform(-1, 1, (2, 6, 3, 24, 40)).astype(np.float32)).cuda()
    ori = visualize.concat_views(visualize.camera_views_u8(px))
    gen = [visualize.concat_views(torch.from_numpy(rng.random((2, 6, 24, 40, 3), dtype=np.float32)).cuda())
           for _ in range(2)]
    layer = lambda: visualize.concat_views(torch.from_numpy(rng.integers(0, 256, (2, 6, 24, 40, 4), dtype=np.uint8)).cuda())
    ori_box, gen_box = layer(), [layer(), layer()]
    paths = visualize.save_run_images(tmp_path, 4, maps, ori, ori_box, gen, gen_box)
    names = [f"{n}_{k}.png" for n in (4, 5) for k in ("map", "ori", "gen0", "gen1", "ori_box", "gen0_box", "gen1_box")]
    assert [os.path.basename(p) for p in paths] == names and sorted(os.listdir(tmp_path)) == sorted(names)
    want = {"4_map.png": O.visualize_map(demo[0], visualize.NUSCENES_MAP_CLASSES, visualize.NUSCENES_OBJECT_CLASSES, 400,
                                         fake_legend)[0],
            "5_ori.png": O.concat_6_views(O.m11_to_u8(px[1].cpu().numpy())),
            "4_gen1.png": gen[1][0].cpu().numpy(), "5_gen0_box.png": gen_box[0][1].cpu().numpy()}
    for name, a in want.items():
        ref = tmp_path.parent / f"pillow_{name}"
        Image.fromarray(np.ascontiguousarray(a)).save(ref)
        assert (tmp_path / name).read_bytes() == ref.read_bytes(), name
