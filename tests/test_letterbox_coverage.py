"""The case table of tests/letterbox_cases.py reaches every letterbox kernel instance, tile-kernel branch, selection
edge and geometry edge (host logic, no GPU needed), and its geometry is the restatement's."""
import numpy as np

from letterbox_cases import CASES, geometry, letterbox_paths
from oracle import restate as R

REQUIRED_PATHS = (
    # the NCHW kernel: the 24 instances launch_src can launch
    {f"nchw {s} {m} -> {d}" for s in ("u8", "f32", "f16", "bf16") for m in ("chw", "hwc") for d in ("f32", "f16", "bf16")}
    # the generic space-to-depth kernel
    | {f"s2d {s} {m} -> {d}" for s in ("f32", "f16", "bf16") for m in ("chw", "hwc") for d in ("f16", "bf16")}
    # the tile kernel's branches
    | {f"tile {m} -> {d}: {b}" for m in ("chw", "hwc") for d in ("f16", "bf16")
       for b in ("copy", "staged identity", "staged", "direct", "fill", "staged + direct in one launch")}
    # the identity kernel
    | {"identity -> f16", "identity -> bf16", "identity: W2 % 64 != 0"}
    # kernel selection and chunked launches
    | {"canvas-size uint8 at an odd byte offset -> tile kernel",
       "canvas-size uint8 batch with a resized image -> tile kernel",
       "several launches, kernel differs by chunk",
       "nchw kernel at img0 > 0", "s2d kernel at img0 > 0", "tile kernel at img0 > 0", "identity kernel at img0 > 0"}
    # geometry
    | {"up-scale from 1x1", "up-scale from 7x9", "up-scale from 61x117", "one axis at ratio 1, the other resized",
       "639 trap", "fixed_shape, asymmetric padding", "odd NCHW canvas",
       "s2d: H2 % 8 != 0", "tile: H2 % 8 != 0", "tile: W2 % 64 != 0", "fill_color 0", "fill_color 255"}
    # rejection: the space-to-depth canvas has no fp32 form
    | {"reject s2d f32 from u8", "reject s2d f32 from f32"}
)


def test_case_names_are_unique():
    names = [c.name for c in CASES]
    assert len(names) == len(set(names))


def test_geometry_is_the_restatements():
    f32 = np.float32
    for c in CASES:
        geoms, (Hb, Wb) = geometry(c)
        sizes = [R.resize_shape(h, w, c.min_size, c.max_size) for h, w in c.sizes]
        assert [(g.src_h, g.src_w) for g in geoms] == list(c.sizes), c.name
        assert [(g.new_h, g.new_w) for g in geoms] == sizes, c.name
        assert (Hb, Wb) == R.batch_shape(sizes, c.size_divisible, c.fixed_shape), c.name
        assert [(g.top, g.left) for g in geoms] == [R.pad_offsets(Hb, Wb, nh, nw) for nh, nw in sizes], c.name
        # the kernels' ratios are ATen's area_pixel_compute_scale: float(in) / float(out)
        assert all(f32(g.ratio_h) == f32(h) / f32(nh) and f32(g.ratio_w) == f32(w) / f32(nw)
                   for g, (h, w), (nh, nw) in zip(geoms, c.sizes, sizes)), c.name


def test_every_path_is_reached():
    seen = {}
    for c in CASES:
        geoms, (Hb, Wb) = geometry(c)
        for p in letterbox_paths(c, geoms, Hb, Wb):
            seen.setdefault(p, []).append(c.name)
    print(f"letterbox path coverage: {len(REQUIRED_PATHS & set(seen))} / {len(REQUIRED_PATHS)} required paths, "
          f"{len(CASES)} cases")
    for p in sorted(REQUIRED_PATHS):
        print(f"  {p}: " + (f"{seen[p][0]}" + (f" (+{len(seen[p]) - 1})" if len(seen[p]) > 1 else "")
                            if p in seen else "MISSING"))
    assert REQUIRED_PATHS <= set(seen), sorted(REQUIRED_PATHS - set(seen))
