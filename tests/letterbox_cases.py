"""One case table for the letterbox kernels (csrc/letterbox.cu).

A `Case` describes one `_C.letterbox` call: the source images (sizes, dtype, memory form), the geometry options of
YOLOTransform (min_size / max_size, size_divisible, fixed_shape, fill_color) and the destination (NCHW fp32 / fp16 /
bf16 or the stem's space-to-depth S2D16 fp16 / bf16 canvas).  `letterbox_paths` names, on the host, the kernels and
branches the call takes: it mirrors the dispatch of `yb_letterbox_strided` / `launch_src` / `launch_typed` and the
per-tile staging decision of `letterbox_s2d_tile_kernel`, with `src_coord`'s fp32 arithmetic.
tests/test_letterbox_coverage.py checks, without a GPU, that the table reaches every required path;
tests/test_gpu_letterbox_paths.py runs every case and compares it bit for bit with `oracle.restate.letterbox`.
"""
import dataclasses
import functools
from typing import List, Optional, Tuple

import numpy as np
import torch

from jpeg_corpus import photo
from oracle import restate as R
from yolort_b200 import _C

f32 = np.float32

DTYPES = {"u8": torch.uint8, "f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}

# csrc/letterbox.cu constants
MAX_IMAGES_PER_LAUNCH = 64      # kMaxImagesPerLaunch
TILE_Y, TILE_X = 8, 64          # kTileY, kTileX: space-to-depth pixels per tile (16 x 128 canvas pixels)
TILE_SMEM = 40 * 1024           # kTileSmem
TILE_MAX_LINES = 3 * 40         # kTileMaxLines


@dataclasses.dataclass(frozen=True)
class Case:
    name: str
    sizes: Tuple[Tuple[int, int], ...]      # (h, w) of each source image
    src: str = "u8"                         # u8 | f32 | f16 | bf16
    mem: str = "chw"                        # chw: contiguous [3,h,w]; hwc: [h,w,3].permute(2,0,1);
    #                                         packed: contiguous [3,h,w] views, back to back in one buffer
    offset: int = 0                         # packed: byte offset of the first image in the buffer
    layout: str = "s2d"                     # nchw | s2d
    dtype: str = "f16"                      # destination: f32 | f16 | bf16 (s2d + f32 is rejected)
    min_size: float = 64.0
    max_size: float = 64.0
    size_divisible: int = 32
    fixed_shape: Optional[Tuple[int, int]] = None
    fill_color: int = 114
    seed: int = 0

    @property
    def layout_code(self) -> int:
        return _C.YB_LAYOUT_NCHW if self.layout == "nchw" else _C.YB_LAYOUT_S2D16


def geometry(case: Case):
    """(geoms, (Hb, Wb)) from the library's host-only geometry (what YOLOTransform.geometry returns)."""
    return _C.letterbox_geometry(case.sizes, case.min_size, case.max_size, case.size_divisible, case.fixed_shape)


def byte_offsets(case: Case) -> List[int]:
    """Byte offset of each image's first element from a 512-byte aligned allocation (0 for separate tensors)."""
    if case.mem != "packed":
        return [0] * len(case.sizes)
    es = torch.empty((), dtype=DTYPES[case.src]).element_size()
    out, o = [], case.offset
    for h, w in case.sizes:
        out.append(o)
        o += 3 * h * w * es
    return out


def reads_hwc(case: Case) -> bool:
    """_C.letterbox reads the batch in place as HWC only when every image is an HWC view (_C._is_hwc_view: a 1 x 1
    image is not one), otherwise as planar CHW."""
    return case.mem == "hwc" and all(h > 1 or w > 1 for h, w in case.sizes)


# ---- host mirror of the dispatch ------------------------------------------------------------------------------------
def src_coord(d: int, ratio: float, size: int) -> Tuple[int, int]:
    """letterbox.cu `src_coord` (lines 65-75) in fp32: the two source indices of canvas offset `d`."""
    real = f32(f32(ratio) * f32(f32(d) + f32(0.5))) - f32(0.5)
    if real < f32(0.0):
        real = f32(0.0)
    i0 = min(int(real), size - 1)
    return i0, i0 + (1 if i0 < size - 1 else 0)


def _is_identity(g) -> bool:
    return g.new_h == g.src_h and g.new_w == g.src_w


@functools.lru_cache(maxsize=None)
def _weights(out_size: int, in_size: int) -> np.ndarray:
    return R._axis_coords(out_size, in_size)[2]


def _informative(g, cy0: int, cy1: int, cx0: int, cx1: int) -> bool:
    """Some row weight and some column weight of the tile's pixels is neither 0 nor 1/2: at 0 the second tap is
    unused, and at 1/2 the two taps weigh the same, so a swapped or misplaced weight would change no value (exact 2x,
    4x, 6x down-scales have only such weights)."""
    ly = _weights(g.new_h, g.src_h)[cy0 - g.top:cy1 - g.top + 1]
    lx = _weights(g.new_w, g.src_w)[cx0 - g.left:cx1 - g.left + 1]
    return bool(np.any((ly != 0) & (ly != 0.5)) and np.any((lx != 0) & (lx != 0.5)))


def tile_staging_bytes(geoms, hwc: bool) -> int:
    """launch_typed (lines 451-460): the dynamic shared memory of a tile-kernel launch over `geoms`."""
    need = 0
    for g in geoms:
        rows = int(f32(2 * TILE_Y) * f32(g.ratio_h)) + 3
        cols = int(f32(2 * TILE_X) * f32(g.ratio_w)) + 3
        line_bytes = 3 * cols if hwc else cols
        need = max(need, (rows if hwc else 3 * rows) * ((line_bytes + 30) // 16 * 16))
    need = min(need, TILE_SMEM)
    return (need + 1023) // 1024 * 1024


def tile_branch(g, hwc: bool, Hb: int, Wb: int, X0: int, Y0: int, need: int) -> str:
    """letterbox_s2d_tile_kernel's branch for the tile at space-to-depth pixel (Y0, X0) of image `g`: `any` (lines
    281-283), the staged rectangle and its fit (285-303), the copy test (306-307) and the sampler choice (347-368).
    A resized tile whose weights are all 0 or 1/2 gets its own name (see `_informative`)."""
    cy0, cy1 = max(2 * Y0, g.top), min(min(2 * (Y0 + TILE_Y), Hb), g.top + g.new_h) - 1
    cx0, cx1 = max(2 * X0, g.left), min(min(2 * (X0 + TILE_X), Wb), g.left + g.new_w) - 1
    if not (cy0 <= cy1 and cx0 <= cx1):
        return "fill"
    ident = _is_identity(g)
    if ident:
        y_lo, y_hi, x_lo, x_hi = cy0 - g.top, cy1 - g.top, cx0 - g.left, cx1 - g.left
    else:
        y_lo = src_coord(cy0 - g.top, g.ratio_h, g.src_h)[0]
        y_hi = src_coord(cy1 - g.top, g.ratio_h, g.src_h)[1]
        x_lo = src_coord(cx0 - g.left, g.ratio_w, g.src_w)[0]
        x_hi = src_coord(cx1 - g.left, g.ratio_w, g.src_w)[1]
    rows, cols = y_hi - y_lo + 1, x_hi - x_lo + 1
    line_bytes = 3 * cols if hwc else cols
    pitch = (line_bytes + 15 + 15) // 16 * 16
    lines = rows if hwc else 3 * rows
    staged = lines <= TILE_MAX_LINES and lines * pitch <= need
    if ident:
        if not staged:
            return "direct identity"
        copy = (cy0, cx0, cy1, cx1) == (2 * Y0, 2 * X0, 2 * (Y0 + TILE_Y) - 1, 2 * (X0 + TILE_X) - 1)
        return "copy" if copy else "staged identity"
    return ("staged" if staged else "direct") + ("" if _informative(g, cy0, cy1, cx0, cx1) else " (weights 0, 1/2 only)")


def launches(case: Case, geoms, Hb: int, Wb: int) -> List[Tuple[str, int, int]]:
    """(kernel, img0, count) of every launch: yb_letterbox_strided's chunks of kMaxImagesPerLaunch images (lines
    674-675) and launch_src / launch_typed's kernel choice per chunk (lines 428-466, 474-486)."""
    hwc = reads_hwc(case)
    offs = byte_offsets(case)
    n = len(case.sizes)
    out = []
    for img0 in range(0, n, MAX_IMAGES_PER_LAUNCH):
        count = min(n - img0, MAX_IMAGES_PER_LAUNCH)
        if case.layout == "s2d" and case.dtype == "f32":
            kernel = "reject"
        elif case.layout == "nchw":
            kernel = "nchw"
        elif case.src == "u8":
            # the identity kernel (lines 433-446): planar sources, every image the whole canvas, 2-byte aligned
            identity = not hwc and Hb % 2 == 0 and Wb % 2 == 0 and all(
                (g.src_h, g.src_w, g.new_h, g.new_w, g.top, g.left) == (Hb, Wb, Hb, Wb, 0, 0) and offs[j] % 2 == 0
                for j, g in enumerate(geoms[img0:img0 + count], img0))
            kernel = "identity" if identity else "tile"
        else:
            kernel = "s2d"
        out.append((kernel, img0, count))
    return out


def _tiles(Hb: int, Wb: int):
    for Y0 in range(0, Hb // 2, TILE_Y):
        for X0 in range(0, Wb // 2, TILE_X):
            yield Y0, X0


def letterbox_paths(case: Case, geoms, Hb: int, Wb: int) -> set:
    """Names of the kernel instances, tile branches, selection edges and geometry edges this case reaches."""
    hwc = reads_hwc(case)
    lay = "hwc" if hwc else "chw"
    geoms = list(geoms)
    paths = set()
    runs = launches(case, geoms, Hb, Wb)
    kernels = {k for k, _, _ in runs}
    if "reject" in kernels:
        return {f"reject s2d f32 from {case.src}"}
    for kernel, img0, count in runs:
        chunk = geoms[img0:img0 + count]
        if img0 > 0:
            paths.add(f"{kernel} kernel at img0 > 0")
        if kernel in ("nchw", "s2d"):
            paths.add(f"{kernel} {case.src} {lay} -> {case.dtype}")
        elif kernel == "identity":
            paths.add(f"identity -> {case.dtype}")
        else:
            need = tile_staging_bytes(chunk, hwc)
            branches = {tile_branch(g, hwc, Hb, Wb, X0, Y0, need) for g in chunk for Y0, X0 in _tiles(Hb, Wb)}
            paths.update(f"tile {lay} -> {case.dtype}: {b}" for b in branches)
            if any(b.startswith("staged") or b == "copy" for b in branches) and any(b.startswith("direct") for b in branches):
                paths.add(f"tile {lay} -> {case.dtype}: staged + direct in one launch")
            canvas_ident = [(g.src_h, g.src_w, g.top, g.left) == (Hb, Wb, 0, 0) and _is_identity(g) for g in chunk]
            if not hwc and all(canvas_ident) and any(o % 2 for o in byte_offsets(case)[img0:img0 + count]):
                paths.add("canvas-size uint8 at an odd byte offset -> tile kernel")
            if not hwc and any(canvas_ident) and not all(canvas_ident):
                paths.add("canvas-size uint8 batch with a resized image -> tile kernel")
    if len(runs) > 1 and len(kernels) > 1:
        paths.add("several launches, kernel differs by chunk")
    # geometry edges
    H2, W2 = Hb // 2, Wb // 2
    if case.layout == "nchw" and (Hb % 2 or Wb % 2):
        paths.add("odd NCHW canvas")
    for k, rows, cols in (("s2d", 8, 128), ("tile", TILE_Y, TILE_X), ("identity", 1, 64)):
        if k in kernels and case.layout == "s2d":
            if H2 % rows:
                paths.add(f"{k}: H2 % {rows} != 0")
            if W2 % cols:
                paths.add(f"{k}: W2 % {cols} != 0")
    for (h, w), g in zip(case.sizes, geoms):
        if g.new_h > h and g.new_w > w:
            paths.add(f"up-scale from {h}x{w}")
        if (g.new_h == h) != (g.new_w == w):
            paths.add("one axis at ratio 1, the other resized")
        if case.max_size == 640 and 639 in (g.new_h, g.new_w):
            paths.add("639 trap")
        if case.fixed_shape is not None and (Hb - g.new_h - g.top != g.top or Wb - g.new_w - g.left != g.left):
            paths.add("fixed_shape, asymmetric padding")
        if (g.new_h, g.new_w) != (Hb, Wb) and case.fill_color in (0, 255):
            paths.add(f"fill_color {case.fill_color}")
    return paths


def pixel_path(case: Case, geoms, Hb: int, Wb: int, n: int, y: int, x: int) -> str:
    """The launch and (tile kernel) branch that wrote canvas pixel (y, x) of image n: for failure messages."""
    geoms = list(geoms)
    for kernel, img0, count in launches(case, geoms, Hb, Wb):
        if img0 <= n < img0 + count:
            where = f"{kernel} kernel, launch img0={img0} count={count}"
            if kernel == "tile":
                need = tile_staging_bytes(geoms[img0:img0 + count], reads_hwc(case))
                Y0, X0 = (y // 2) // TILE_Y * TILE_Y, (x // 2) // TILE_X * TILE_X
                where += f", tile (Y0={Y0}, X0={X0}) {tile_branch(geoms[n], reads_hwc(case), Hb, Wb, X0, Y0, need)}"
            return where
    raise IndexError(n)


# ---- images -----------------------------------------------------------------------------------------------------------
def _content(h: int, w: int, src: str, seed: int) -> np.ndarray:
    """[h, w, 3]: smooth structure with saturated blocks (jpeg_corpus.photo) plus uniform noise on an eighth of the
    values, so that every byte value occurs; float sources span [-2, 3]."""
    r = np.random.default_rng(seed + 7919)
    a = photo(h, w, seed)
    noise = r.random((h, w, 3)) < 0.125
    a[noise] = r.integers(0, 256, int(noise.sum()), dtype=np.uint8)
    if src == "u8":
        return a
    return a.astype(np.float32) * f32(5.0 / 255.0) - f32(2.0) + r.uniform(-0.02, 0.02, (h, w, 3)).astype(np.float32)


def make_images(case: Case, device) -> Tuple[List[torch.Tensor], List[torch.Tensor]]:
    """(images on `device` in the case's memory form, the same values as CPU [3,h,w] tensors for the reference)."""
    dt = DTYPES[case.src]
    hwc = [torch.from_numpy(_content(h, w, case.src, case.seed * 1009 + i)).to(dt)
           for i, (h, w) in enumerate(case.sizes)]
    ref = [t.permute(2, 0, 1) for t in hwc]
    if case.mem == "hwc":
        return [t.to(device).permute(2, 0, 1) for t in hwc], ref
    if case.mem == "chw":
        return [t.contiguous().to(device) for t in ref], ref
    es = torch.empty((), dtype=dt).element_size()
    assert case.offset % es == 0, "a packed view starts on an element boundary"
    flat = torch.cat([torch.zeros(case.offset // es, dtype=dt)] + [t.reshape(-1) for t in
                                                                   (r.contiguous() for r in ref)] + [torch.zeros(8, dtype=dt)])
    buf = flat.to(device)
    views, o = [], case.offset // es
    for h, w in case.sizes:
        views.append(buf[o:o + 3 * h * w].view(3, h, w))
        o += 3 * h * w
    return views, ref


# ---- the table ----------------------------------------------------------------------------------------------------------
def _cases() -> List[Case]:
    out = []
    seed = 0

    def add(**kw):
        nonlocal seed
        seed += 1
        out.append(Case(seed=seed, **kw))

    small = ((50, 70), (64, 64), (33, 20))     # 64 x 64 canvas: a down-scale, an identity, an up-scale
    # the NCHW kernel: every source dtype x source layout x destination dtype (the 24 instances launch_src can launch)
    for src in ("u8", "f32", "f16", "bf16"):
        for mem in ("chw", "hwc"):
            for dt in ("f32", "f16", "bf16"):
                add(name=f"nchw {src} {mem} -> {dt}", sizes=small, src=src, mem=mem, layout="nchw", dtype=dt)
    # the generic space-to-depth kernel: float sources
    for src in ("f32", "f16", "bf16"):
        for mem in ("chw", "hwc"):
            for dt in ("f16", "bf16"):
                add(name=f"s2d {src} {mem} -> {dt}", sizes=small, src=src, mem=mem, dtype=dt)
    # the tile kernel: a copy image (the whole canvas), an identity image with padding (partial edge tiles and
    # fill-only tiles), a ~1.95x down-scale (staged) and a ~3.9x down-scale (direct) in one launch
    for mem in ("chw", "hwc"):
        for dt in ("f16", "bf16"):
            add(name=f"tile {mem} -> {dt} all branches", sizes=((256, 256), (200, 256), (500, 410), (1000, 1000)),
                mem=mem, dtype=dt, min_size=256, max_size=256)
    # camera frames: all-direct (1080p, 4K) and one image whose tiles split between staged and direct (1700 x 956)
    add(name="1080p hwc -> f16", sizes=((1080, 1920),), mem="hwc", min_size=640, max_size=640)
    add(name="1920x1080 chw -> bf16", sizes=((1920, 1080),), dtype="bf16", min_size=640, max_size=640)
    add(name="1700x956 chw -> f16 staged and direct tiles", sizes=((1700, 956),), min_size=640, max_size=640)
    add(name="1700x956 hwc -> bf16 staged and direct tiles", sizes=((1700, 956),), mem="hwc", dtype="bf16",
        min_size=640, max_size=640)
    add(name="4K hwc -> bf16", sizes=((2160, 3840),), mem="hwc", dtype="bf16", min_size=640, max_size=640)
    # the identity kernel (canvas-size planar uint8 batches)
    add(name="identity 640 -> f16", sizes=((640, 640),) * 2, min_size=640, max_size=640)
    add(name="identity 96x160 -> bf16 (W2 = 80)", sizes=((96, 160),) * 3, dtype="bf16", min_size=96, max_size=160)
    add(name="identity 96x160 -> f16 packed at byte 2", sizes=((96, 160),) * 2, mem="packed", offset=2,
        min_size=96, max_size=160)
    # selection edges
    add(name="canvas-size uint8 at byte 1 -> tile copy", sizes=((96, 160),) * 2, mem="packed", offset=1,
        min_size=96, max_size=160)
    add(name="canvas-size uint8 + one resized -> tile", sizes=((64, 64), (64, 64), (128, 100)), dtype="bf16")
    add(name="70 images: identity chunk then tile chunk", sizes=((64, 64),) * 64 + ((100, 80), (30, 64)) * 3,
        dtype="bf16")
    add(name="66 images: tile chunk then identity chunk", sizes=((50, 70), (64, 64)) * 32 + ((64, 64),) * 2)
    add(name="66 images nchw u8 hwc -> f16", sizes=((50, 70), (64, 64), (33, 20)) * 22, mem="hwc", layout="nchw")
    add(name="66 images s2d f16 -> bf16", sizes=((50, 70), (64, 64), (33, 20)) * 22, src="f16", dtype="bf16")
    # geometry edges
    add(name="up-scale 1x1 7x9 61x117 -> 640 s2d f16", sizes=((1, 1), (7, 9), (61, 117)), min_size=640, max_size=640)
    add(name="up-scale 1x1 7x9 61x117 hwc -> 640 s2d bf16", sizes=((1, 1), (7, 9), (61, 117)), mem="hwc",
        dtype="bf16", min_size=640, max_size=640)
    add(name="up-scale 7x9 61x117 f32 hwc -> 640 nchw f32", sizes=((7, 9), (61, 117)), src="f32", mem="hwc",
        layout="nchw", dtype="f32", min_size=640, max_size=640)
    add(name="ratio 1 on h only (599x600 at 600/1000) hwc -> bf16", sizes=((599, 600),), mem="hwc", dtype="bf16",
        min_size=600, max_size=1000)
    add(name="ratio 1 on h only (8x89 at 64/100) f32 -> nchw f32", sizes=((8, 89), (20, 30)), src="f32",
        layout="nchw", dtype="f32", min_size=64, max_size=100)
    add(name="639 trap -> nchw f32", sizes=((800, 600), (480, 640)), layout="nchw", dtype="f32",
        min_size=640, max_size=640)
    add(name="639 trap -> s2d f16", sizes=((800, 600), (480, 640)), min_size=640, max_size=640)
    add(name="fixed_shape 672x704 asymmetric -> s2d bf16", sizes=((800, 600),), dtype="bf16", min_size=640,
        max_size=640, fixed_shape=(672, 704))
    add(name="fixed_shape 75x97 bf16 -> nchw f16", sizes=((50, 70), (33, 20)), src="bf16", layout="nchw",
        min_size=64, max_size=64, fixed_shape=(75, 97))
    add(name="odd canvas 45x64 (size_divisible 1) -> nchw bf16", sizes=((70, 101), (50, 70)), layout="nchw",
        dtype="bf16", size_divisible=1)
    add(name="odd canvas 44x63 (size_divisible 1) f16 hwc -> nchw f32", sizes=((70, 101),), src="f16", mem="hwc",
        layout="nchw", dtype="f32", size_divisible=1)
    add(name="canvas 100x150 -> tile (H2 = 50, W2 = 75)", sizes=((100, 150), (200, 300)), min_size=150,
        max_size=150, size_divisible=2)
    add(name="canvas 100x150 f32 -> s2d bf16 (H2 = 50, W2 = 75)", sizes=((100, 150), (200, 300)), src="f32",
        dtype="bf16", min_size=150, max_size=150, size_divisible=2)
    add(name="fill 0 -> tile f16", sizes=((50, 70), (64, 64), (200, 40)), fill_color=0)
    add(name="fill 255 -> tile bf16 hwc", sizes=((50, 70), (64, 64), (200, 40)), mem="hwc", dtype="bf16",
        fill_color=255)
    add(name="fill 0 f32 -> nchw f32", sizes=small, src="f32", layout="nchw", dtype="f32", fill_color=0)
    # rejection: the space-to-depth canvas is fp16 / bf16 only
    add(name="reject s2d f32 from u8", sizes=small, dtype="f32")
    add(name="reject s2d f32 from f32", sizes=small, src="f32", dtype="f32")
    return out


CASES = _cases()
