"""Map images and mosaics on the CPU: the numpy restatement (oracle/map_visualizer.py) against the reference's own images
(tests/golden/map_visualizer.pt), visualize.py's host logic through the CPU restatement of its kernels, and the argument
checks, which all come before anything is returned or written."""
import hashlib
import importlib.util
import os

import numpy as np
import pytest
import torch
from PIL import Image

from magicdrive_b200 import visualize
from oracle import map_visualizer as O
from oracle.make_golden_map_visualizer import REF, fake_legend, load
from tests import image_ops_emulator, visualize_ops_emulator
from tests.common import GOLDEN

FX = load(os.path.join(GOLDEN, "map_visualizer.pt"))
MAPS = {c["name"]: c for c in FX["maps"]}


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


@pytest.fixture
def emulated(monkeypatch):
    image_ops_emulator.install(monkeypatch)
    visualize_ops_emulator.install(monkeypatch)


@pytest.mark.parametrize("name", sorted(MAPS))
def test_oracle_equals_reference_map_image(name):
    c = MAPS[name]
    img, names = O.visualize_map(c["map"], FX["map_classes"], FX["object_classes"], c["target_size"], fake_legend)
    assert sorted(names) == c["legend_names"] and c["legend_size"] == c["target_size"]
    assert img.shape == tuple(c["out_shape"]) and _sha(img) == c["sha256"]
    if "out" in c:
        assert np.array_equal(img, c["out"])


def test_fixture_covers_both_legend_placements_and_the_identity_resize():
    assert {c["right"] for c in FX["maps"]} == {True, False}
    assert MAPS["identity400@400"]["map"].shape[-1] == 400 and MAPS["demo0@150"]["out_shape"][1] == 150


@pytest.mark.parametrize("i", range(len(FX["mosaics"])))
def test_oracle_equals_reference_mosaic(i):
    c = FX["mosaics"][i]
    assert np.array_equal(O.concat_6_views(c["views"], c["oneline"]), c["out"])


def test_oracle_equals_reference_camera_views():
    m = FX["m11"]
    assert m["n_demo_values"] == 256
    assert np.array_equal(O.m11_to_u8(m["x"].numpy()), m["out"].numpy())


@pytest.mark.parametrize("name", ["demo0@400", "demo3@800", "demo0@150", "seeded18@400", "seeded26@400", "zeros18@400",
                                  "identity400@400"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.uint8, torch.bool])
def test_host_logic_equals_reference(emulated, name, dtype):
    """visualize_maps with its kernels restated on the CPU, a batch of the case's map and its transpose."""
    c = MAPS[name]
    m = torch.from_numpy(c["map"].copy())
    batch = torch.stack([m, m.transpose(1, 2)]).to(dtype)
    calls = []

    def legend(names, size):
        calls.append(names)
        return fake_legend(names, size)

    out = visualize.visualize_maps(batch, FX["map_classes"], FX["object_classes"], c["target_size"], legend=legend)
    assert out[0].shape == tuple(c["out_shape"]) and _sha(out[0].numpy()) == c["sha256"]
    want, names = O.visualize_map(batch[1].numpy().astype(np.uint8), FX["map_classes"], FX["object_classes"],
                                  c["target_size"], fake_legend)
    assert np.array_equal(out[1].numpy(), want)
    assert len(calls) == len(set(calls)) and set(calls) == {frozenset(c["legend_names"]), names}


def test_each_legend_is_drawn_once_per_process(emulated, monkeypatch):
    """The default legend is drawn once per process for each (names, size); a caller's callable once while it is the
    last one passed, and a fresh callable per call is drawn anew without the caches growing."""
    m = torch.from_numpy(MAPS["demo1@400"]["map"].copy()).expand(5, -1, -1, -1)
    calls = []

    def legend(names, size):
        calls.append((names, size))
        return fake_legend(names, size)

    monkeypatch.setattr(visualize, "_LEGENDS", {})
    monkeypatch.setattr(visualize, "_DEVICE_LEGENDS", {})
    monkeypatch.setattr(visualize, "show_legend", legend)
    for _ in range(3):
        visualize.visualize_maps(m)
    visualize.visualize_maps(m, target_size=800)
    assert len(calls) == 2 and calls[0][1] == 400 and calls[1][1] == 800
    del calls[:]
    n_host, n_dev = len(visualize._LEGENDS), len(visualize._DEVICE_LEGENDS)
    for _ in range(3):
        visualize.visualize_maps(m, legend=legend)
    assert len(calls) == 1
    for _ in range(3):
        visualize.visualize_maps(m, legend=lambda names, size: legend(names, size))
    assert len(calls) == 4 and (len(visualize._LEGENDS), len(visualize._DEVICE_LEGENDS)) == (n_host, n_dev)
    assert len(visualize._CALLER[1]) == 1 and len(visualize._CALLER[2]) == 1


def test_cached_legend_is_a_copy(emulated, monkeypatch):
    a = np.full((50, 400, 3), 9, np.uint8)
    monkeypatch.setattr(visualize, "_LEGENDS", {})
    monkeypatch.setattr(visualize, "_DEVICE_LEGENDS", {})
    monkeypatch.setattr(visualize, "show_legend", lambda names, size: a)
    m = torch.from_numpy(MAPS["demo1@400"]["map"].copy())[None]
    first = visualize.visualize_maps(m)[0].clone()
    a[:] = 0  # the caller reuses its array
    visualize._DEVICE_LEGENDS.clear()
    assert torch.equal(visualize.visualize_maps(m)[0], first)


def error_cases():
    """Maps on which the reference raises, and which error it raises first: render_static fails at the first pixel, in
    raster order, where get_color_by_priority does (the rank lookup before the colour's, at every pixel with a static
    class, under an object or not), before render_dynamic looks up the object classes' colours.  -> {name: (maps fp32
    (B, 18, 24, 24), map_classes, object_classes, exception, message)}."""
    ranked = list(visualize.NUSCENES_MAP_CLASSES[:6])
    objs = list(visualize.NUSCENES_OBJECT_CLASSES)
    van = objs[:9] + ["van"]
    cases = {}

    def maps(*pixels, B=1):
        m = torch.zeros(B, 18, 24, 24)
        for b, c, y, x in pixels:
            m[b, c, y, x] = 1
        return m

    # "divider" ranks above drivable_area and has no colour; it wins only under a car
    cases["colourless_under_object"] = (maps((0, 0, 3, 3), (0, 7, 4, 5), (0, 8, 4, 5), (0, 0, 4, 5)),
                                        ranked + ["lane_divider", "divider"], objs, KeyError, "divider")
    both = ranked + ["lane", "divider"]  # lane: no rank; divider: no colour
    cases["colour_error_first"] = (maps((0, 7, 2, 3), (0, 6, 5, 5)), both, objs, KeyError, "divider")
    cases["rank_error_first"] = (maps((0, 7, 2, 3), (0, 6, 1, 20)), both, objs, ValueError, "'lane' is not in list")
    cases["same_pixel"] = (maps((0, 7, 2, 3), (0, 6, 2, 3)), both, objs, ValueError, "'lane' is not in list")
    cases["static_before_object_colour"] = (maps((0, 6, 9, 9)), ranked + ["lane", "walkway"], van, ValueError,
                                            "'lane' is not in list")
    cases["object_colour"] = (maps((0, 0, 9, 9)), ranked + ["road_block", "walkway"], van, KeyError, "van")
    cases["first_map_first"] = (maps((1, 6, 0, 0), B=2), ranked + ["lane", "walkway"], van, KeyError, "van")
    return cases


ERRORS = error_cases()


@pytest.mark.parametrize("name", sorted(ERRORS))
def test_errors_in_the_reference_order(emulated, name):
    m, classes, objs, exc, msg = ERRORS[name]
    with pytest.raises(exc, match=msg):
        for b in range(m.shape[0]):  # the reference, one map after another
            O.visualize_map(m[b].numpy(), classes, objs, 48, fake_legend)
    with pytest.raises(exc, match=msg):
        visualize.visualize_maps(m, classes, objs, 48, legend=fake_legend)


@pytest.mark.skipif(not os.path.exists(os.path.join(REF, "magicdrive", "runner", "map_visualizer.py")),
                    reason="needs the reference tree")
@pytest.mark.parametrize("name", sorted(ERRORS))
def test_error_cases_are_the_reference_errors(name):
    """The reference's own visualize_map (taken as the fixture script takes it) raises the same error."""
    from types import SimpleNamespace

    from oracle.make_golden_map_visualizer import reference_namespace
    m, classes, objs, exc, msg = ERRORS[name]
    ns = reference_namespace([])
    cfg = SimpleNamespace(dataset=SimpleNamespace(map_classes=classes, object_classes=objs))
    with pytest.raises(exc, match=msg):
        for b in range(m.shape[0]):
            ns["visualize_map"](cfg, m[b], target_size=48)


def _maps(C=18, H=24, seed=0):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand((2, C, H, H), generator=g) < 0.2).float()


@pytest.mark.parametrize("bad", [2.0, 0.5, -1.0, float("nan"), 1e-40])
def test_non_binary_map_raises(emulated, bad):
    m = _maps()
    m[1, 3, 5, 7] = bad
    with pytest.raises(ValueError, match="values other than 0 and 1"):
        visualize.visualize_maps(m, target_size=48, legend=fake_legend)
    m = _maps(C=26)
    m[1, 20, 0, 0] = bad  # an aux layer past the dynamic ones is never read
    visualize.visualize_maps(m, target_size=48, legend=fake_legend)


def test_static_class_missing_from_priority_raises_value_error(emulated):
    classes = list(visualize.NUSCENES_MAP_CLASSES[:7]) + ["lane"]
    m = _maps()
    with pytest.raises(ValueError, match="'lane' is not in list"):
        visualize.visualize_maps(m, classes, legend=fake_legend, target_size=48)
    m[:, 7] = 0  # inactive, it is never looked up
    assert len(visualize.visualize_maps(m, classes, legend=fake_legend, target_size=48)) == 2


def test_chosen_class_without_colour_raises_key_error(emulated):
    classes = list(visualize.NUSCENES_MAP_CLASSES[:7]) + ["divider"]  # in STATIC_PRIORITY, not in COLORS
    m = _maps()
    m[:, 5:7] = 0  # nothing ranked above "divider"
    with pytest.raises(KeyError, match="divider"):
        visualize.visualize_maps(m, classes, legend=fake_legend, target_size=48)
    m[:, 6] = m[:, 7]  # lane_divider wherever divider is: divider is never drawn
    assert len(visualize.visualize_maps(m, classes, legend=fake_legend, target_size=48)) == 2


def test_object_class_without_colour_raises_key_error(emulated):
    with pytest.raises(KeyError, match="van"):
        visualize.visualize_maps(_maps(), object_classes=list(visualize.NUSCENES_OBJECT_CLASSES[:9]) + ["van"],
                                 legend=fake_legend, target_size=48)


def test_shape_and_layer_checks(emulated):
    with pytest.raises(ValueError, match="only square maps"):
        visualize.visualize_maps(torch.zeros(1, 18, 20, 24), legend=fake_legend)
    with pytest.raises(ValueError, match="neither static nor dynamic"):
        visualize.visualize_maps(torch.zeros(1, 8, 20, 20), map_classes=(), object_classes=(), legend=fake_legend)
    with pytest.raises(ValueError):
        visualize.visualize_maps(torch.zeros(1, 8, 20, 20, dtype=torch.int64), legend=fake_legend)
    # 8 channels with classes for 18: the static layers only, as the reference's slices give, so no class is named
    # (and the fake legend of the empty set stands beside the map)
    out = visualize.visualize_maps(torch.zeros(1, 8, 20, 20), legend=fake_legend, target_size=40)
    assert out[0].shape == (40, 40 + 40 // 8, 3)


def test_legend_that_does_not_fit_raises(emulated):
    m = torch.zeros(1, 18, 97, 97)
    assert visualize.resized_side(97, 400) == 399  # int(97 * (400 / 97)): the reference's own rounding
    with pytest.raises(ValueError, match="does not fit"):
        visualize.visualize_maps(m, target_size=400, legend=fake_legend)
    with pytest.raises(ValueError, match="uint8"):
        visualize.visualize_maps(m, target_size=300, legend=lambda n, s: np.zeros((5, s, 3), np.float32))
    # numpy broadcasts a single-row legend across the width, so does visualize_maps
    out = visualize.visualize_maps(m, target_size=400, legend=lambda n, s: np.full((1, 1, 3), 7, np.uint8))
    assert out[0].shape == (400, 399, 3) and bool((out[0][399:] == 7).all())


def test_mosaic_checks(emulated):
    with pytest.raises(ValueError, match="at least 5 views"):
        visualize.concat_views(torch.zeros(1, 4, 8, 8, 3, dtype=torch.uint8))
    with pytest.raises(ValueError, match="at least 2 views"):
        visualize.concat_views(torch.zeros(1, 1, 8, 8, 3, dtype=torch.uint8), oneline=True)
    with pytest.raises(ValueError):
        visualize.concat_views(torch.zeros(1, 6, 8, 8, 4, dtype=torch.float32))
    with pytest.raises(ValueError):
        visualize.camera_views_u8(torch.zeros(1, 6, 4, 8, 8))


@pytest.mark.parametrize("i", range(len(FX["mosaics"])))
def test_mosaic_host_logic_equals_reference(emulated, i):
    c = FX["mosaics"][i]
    out = visualize.concat_views(torch.from_numpy(c["views"].copy())[None], c["oneline"])
    assert np.array_equal(out[0].numpy(), c["out"])


def test_camera_views_host_logic_equals_reference(emulated):
    m = FX["m11"]
    out = visualize.camera_views_u8(m["x"][None, None])
    assert np.array_equal(out[0, 0].numpy(), m["out"].numpy())


def test_save_run_images_writes_the_reference_file_set(emulated, tmp_path):
    maps = visualize.visualize_maps(_maps(), target_size=48, legend=fake_legend)
    rng = np.random.default_rng(3)
    mosaic = lambda c: torch.from_numpy(rng.integers(0, 256, (2, 16, 24, c), dtype=np.uint8))
    ori, ori_box, gen, gen_box = mosaic(3), mosaic(4), [mosaic(3), mosaic(3)], [mosaic(4), mosaic(4)]
    paths = visualize.save_run_images(tmp_path, 10, maps, ori, ori_box, gen, gen_box)
    names = [f"{n}_{k}.png" for n in (10, 11) for k in ("map", "ori", "gen0", "gen1", "ori_box", "gen0_box", "gen1_box")]
    assert [os.path.basename(p) for p in paths] == names and sorted(os.listdir(tmp_path)) == sorted(names)
    want = {"10_map.png": maps[0], "11_ori.png": ori[1], "10_gen1.png": gen[1][0], "11_gen0_box.png": gen_box[0][1]}
    for name, img in want.items():
        ref = tmp_path / f"ref_{name}"
        Image.fromarray(img.numpy()).save(ref)
        assert (tmp_path / name).read_bytes() == ref.read_bytes()


def test_save_run_images_checks_before_writing(tmp_path):
    maps = [torch.zeros(8, 8, 3, dtype=torch.uint8)] * 2
    with pytest.raises(ValueError, match="gen\\[1\\] holds 1 images for 2 maps"):
        visualize.save_run_images(tmp_path, 0, maps, gen=[torch.zeros(2, 8, 8, 3, dtype=torch.uint8),
                                                          torch.zeros(1, 8, 8, 3, dtype=torch.uint8)])
    with pytest.raises(ValueError, match="uint8"):
        visualize.save_run_images(tmp_path, 0, maps, ori=torch.zeros(2, 8, 8, 3))
    assert os.listdir(tmp_path) == []


def test_default_legend_needs_matplotlib(emulated, monkeypatch):
    import builtins
    real_import = builtins.__import__

    def no_matplotlib(name, *a, **k):
        if name.startswith("matplotlib"):
            raise ImportError(f"No module named {name!r}")
        return real_import(name, *a, **k)

    monkeypatch.setattr(builtins, "__import__", no_matplotlib)
    monkeypatch.setattr(visualize, "_LEGENDS", {})
    monkeypatch.setattr(visualize, "_DEVICE_LEGENDS", {})
    with pytest.raises(ImportError, match="matplotlib"):
        visualize.visualize_maps(_maps(), target_size=48)


@pytest.mark.skipif(importlib.util.find_spec("matplotlib") is None or
                    not os.path.exists(os.path.join(REF, "magicdrive", "runner", "map_visualizer.py")),
                    reason="needs matplotlib and the reference tree")
@pytest.mark.parametrize("size", [150, 400, 800])
def test_default_legend_equals_reference_show_legend(size):
    import ast
    import io

    import matplotlib.patches as mpatches
    import matplotlib.pyplot as plt
    ns = {"np": np, "io": io, "Image": Image, "plt": plt, "mpatches": mpatches}
    src = open(os.path.join(REF, "magicdrive", "runner", "map_visualizer.py")).read()
    for node in ast.parse(src).body:
        if getattr(node, "name", None) in ("rgb_to_01range", "show_legend") or \
                isinstance(node, ast.Assign) and getattr(node.targets[0], "id", None) == "COLORS":
            exec(compile(ast.Module([node], []), "map_visualizer.py", "exec"), ns)
    for names in (frozenset({"car"}), frozenset(MAPS["seeded18@400"]["legend_names"]),
                  frozenset(MAPS["demo4@400"]["legend_names"])):
        assert np.array_equal(visualize.show_legend(names, size), ns["show_legend"](set(names), long_edge_size=size))
