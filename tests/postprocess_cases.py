"""One case table for the post-processing kernels (csrc/decode_nms.cu) and the fused decode epilogue of the head
convolutions (`decode_fragment`, csrc/conv_sm90.cu).

A `Case` describes one `yb_nms_begin` / `yb_decode_candidates` / `yb_nms_finish` sequence: the head levels, their
layout (the reference's [N, A, H, W, K] or the plan's NHWC rows), row pitch, base offset and dtype, the anchors and
classes, the logit distribution per image, and the NMS options (score / IoU threshold, semantics, max_det, rescale and
the candidate arena's share per image).  A `FusedCase` describes a plan of 1x1 head convolutions whose epilogue decodes
into a `_C.FusedPost` arena.

`postprocess_paths` names, on the host, the kernels and branches a case takes: it mirrors the kernel choice of
`yb_decode_candidates` (the row kernel's eligibility test), the row kernel's copy and candidate-list branches, and the
NMS kernel's sort, semantics, label-mask, sweep and overflow branches from the reference candidates.
tests/test_postprocess_coverage.py checks, without a GPU, that the tables reach every required path;
tests/test_gpu_postprocess_paths.py runs every case on the GPU and compares the decode stage with `reference` (fp64)
and the NMS stage bit for bit with `oracle.restate.batched_nms` on the kernel's own candidates.
"""
import ctypes
import dataclasses
import functools
from typing import List, Optional, Tuple

import numpy as np
import torch

from oracle import restate as R
from yolort_b200 import _C

DTYPES = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}
ANCHORS4 = [[10, 13, 16, 30, 33, 23, 8, 9], [30, 61, 62, 45, 59, 119, 40, 30], [116, 90, 156, 198, 373, 326, 200, 150],
            [436, 615, 739, 380, 925, 792, 600, 500]]
STRIDES = [8, 16, 32, 64]

# csrc/decode_nms.cu constants
ROW_MAX_BYTES = 512             # kRowMaxBytes
ROW_MAX_EXTENT = 1023           # kRowMaxExtent
ROW_PIXELS, ROW_WARPS = 32, 4   # kRowPixels, kRowWarps: a block takes 128 pixels of one image
ROW_LIST = 512                  # kRowList: block-local candidate list
SWEEP = 512                     # kSweep
MAX_LABEL_MASKS = 256           # kMaxLabelMasks
SMALL_SORT = 4096               # kSmallSort
NMS_THREADS = 512               # kNmsThreads

# A pair whose fp64 score lies within this relative distance of the threshold may go either way on the GPU: expf
# differs from the exact exponential by up to 2 ulp, and the sigmoid and the product round three more times.
SCORE_BAND = 2.0 ** -20


@dataclasses.dataclass(frozen=True)
class Case:
    name: str
    levels: Tuple[Tuple[int, int], ...]      # (H, W) of each level
    layout: str = "nhwc"                     # nhwc: [N, H, W, pitch], channel a * K + k; nahwk: [N, A, H, W, K]
    pitch: int = 256                         # nhwc: elements per pixel row (the plan's head buffers: 256)
    offset: int = 0                          # elements between the 512-byte aligned allocation and the first logit
    dtype: str = "f16"
    anchors: int = 3
    nc: int = 80
    n_images: int = 2
    spread: float = 1.5                      # standard deviation of every logit
    obj_shift: float = -2.0                  # added to the objectness logits
    cls_shift: float = -1.0                  # added to the class logits
    image_shift: Tuple[float, ...] = ()      # added to the objectness logits of image i
    thr: float = 0.25
    iou: float = 0.45
    semantics: int = R.TV_AUTO
    max_det: int = 300
    rescale: bool = False
    cap: int = 16384                         # candidate-arena share per image
    seed: int = 0

    @property
    def K(self) -> int:
        return self.nc + 5

    @property
    def anchors_px(self) -> List[List[float]]:
        return [[float(v) for v in ANCHORS4[i][:2 * self.anchors]] for i in range(len(self.levels))]

    @property
    def strides(self) -> List[int]:
        return STRIDES[:len(self.levels)]

    @property
    def esize(self) -> int:
        return 4 if self.dtype == "f32" else 2


# ---- inputs -------------------------------------------------------------------------------------------------------------
def logits(case: Case) -> List[torch.Tensor]:
    """[N, A, H, W, K] per level, rounded to the case's dtype (CPU)."""
    g = torch.Generator().manual_seed(1000 + case.seed)
    out = []
    for (h, w) in case.levels:
        t = torch.randn(case.n_images, case.anchors, h, w, case.K, generator=g) * case.spread
        t[..., 4] += case.obj_shift
        t[..., 5:] += case.cls_shift
        for i, s in enumerate(case.image_shift):
            t[i, ..., 4] += s
        out.append(t.to(DTYPES[case.dtype]))
    return out


GUARD_LOGIT = 9.0     # pad channels and guard elements: a kernel that read them would find sure candidates


def head_tensors(case: Case, device) -> List[torch.Tensor]:
    """The levels in the case's layout on `device`, each a contiguous view `offset` elements into its allocation."""
    out = []
    for t in logits(case):
        n, a, h, w, k = t.shape
        if case.layout == "nhwc":
            v = torch.full((n, h, w, case.pitch), GUARD_LOGIT, dtype=t.dtype)
            v[..., :a * k] = t.permute(0, 2, 3, 1, 4).reshape(n, h, w, a * k)
        else:
            v = t
        flat = torch.full((case.offset + v.numel() + 64,), GUARD_LOGIT, dtype=t.dtype)
        flat[case.offset:case.offset + v.numel()] = v.reshape(-1)
        out.append(flat.to(device)[case.offset:case.offset + v.numel()].view(v.shape))
    return out


def rescale_params(case: Case) -> Optional[np.ndarray]:
    """[N, 3] (gain, padx, pady) per image: a letterbox of a landscape and a portrait image into the canvas."""
    if not case.rescale:
        return None
    Hb, Wb = case.levels[0][0] * case.strides[0], case.levels[0][1] * case.strides[0]
    sizes = [(int(Hb * 0.6) + 3 * i, Wb + 40 * i) if i % 2 == 0 else (Hb + 17 * i, int(Wb * 0.7)) for i in
             range(case.n_images)]
    return np.array([R.scale_coords_params(Hb, Wb, h, w) for h, w in sizes], dtype=np.float32)


# ---- fp64 reference of the decode ---------------------------------------------------------------------------------------
@dataclasses.dataclass
class Ref:
    scores: np.ndarray      # [N, A_total, nc] fp64
    boxes: np.ndarray       # [N, A_total, 4] fp64 xyxy
    scale: np.ndarray       # [N, A_total] fp64 |cx| + |cy| + w + h: the boxes' rounding scale
    pixel: np.ndarray       # [A_total] flat pixel index (the row kernel's r) of each anchor


def _sig(x):
    return 1.0 / (1.0 + np.exp(-x))


def decode64(levels64: List[np.ndarray], strides, anchors_px) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """restate.decode in fp64 on [N, A, H, W, K] logits: (scores [N, A_total, nc], boxes xyxy, |cx|+|cy|+w+h)."""
    scores, boxes, scale = [], [], []
    for l, t in enumerate(levels64):
        n, a, h, w, k = t.shape
        y = _sig(t)
        gx = np.arange(w, dtype=np.float64).reshape(1, 1, 1, w)
        gy = np.arange(h, dtype=np.float64).reshape(1, 1, h, 1)
        st = float(strides[l])
        anc = np.array(anchors_px[l][:2 * a], dtype=np.float64).reshape(1, a, 1, 1, 2)
        cx = (y[..., 0] * 2.0 - 0.5 + gx) * st
        cy = (y[..., 1] * 2.0 - 0.5 + gy) * st
        wh = (y[..., 2:4] * 2.0) ** 2 * anc
        bw, bh = wh[..., 0], wh[..., 1]
        boxes.append(np.stack((cx - 0.5 * bw, cy - 0.5 * bh, cx + 0.5 * bw, cy + 0.5 * bh), -1).reshape(n, -1, 4))
        scale.append((np.abs(cx) + np.abs(cy) + bw + bh).reshape(n, -1))
        scores.append((y[..., 5:] * y[..., 4:5]).reshape(n, -1, k - 5))
    return np.concatenate(scores, 1), np.concatenate(boxes, 1), np.concatenate(scale, 1)


def pixel_index(levels, anchors: int) -> np.ndarray:
    """Flat pixel index (pix_start[level] + y * W + x) of every flat anchor index (lvl_start + (a * H + y) * W + x)."""
    out, p0 = [], 0
    for h, w in levels:
        out.append(np.tile(p0 + np.arange(h * w), anchors))
        p0 += h * w
    return np.concatenate(out)


@functools.lru_cache(maxsize=None)
def reference(case: Case) -> Ref:
    lv = [t.double().numpy() for t in logits(case)]
    s, b, sc = decode64(lv, case.strides, case.anchors_px)
    return Ref(s, b, sc, pixel_index(case.levels, case.anchors))


def membership(scores64: np.ndarray, thr: float, band: np.ndarray):
    """(sure, ambiguous) boolean masks over [A_total, nc]: pairs over the threshold beyond any rounding, and pairs
    within `band` of it that the kernel may take either way."""
    d = scores64 - np.float64(np.float32(thr))
    amb = np.abs(d) <= band
    return (d > 0) & ~amb, amb


def score_band(case: Case, scores64: np.ndarray) -> np.ndarray:
    return SCORE_BAND * np.maximum(np.float64(np.float32(case.thr)), scores64)


# ---- host mirror of the kernel choice and branches ----------------------------------------------------------------------
def level_strides(case: Case, h: int, w: int) -> Tuple[int, int, int, int]:
    """(stride_n, stride_a, stride_y, stride_x) in elements, as _C._level_struct sets them."""
    a, k = case.anchors, case.K
    if case.layout == "nhwc":
        C = case.pitch
        return h * w * C, k, w * C, C
    return a * h * w * k, h * w * k, w * k, k


def uses_rows(case: Case) -> bool:
    """yb_decode_candidates' `rows` predicate: 16-bit NHWC rows of at most 512 bytes, 16-byte aligned, levels at most
    kRowMaxExtent wide and tall."""
    if case.dtype not in ("f16", "bf16"):
        return False
    for h, w in case.levels:
        sn, sa, sy, sx = level_strides(case, h, w)
        if not (h <= ROW_MAX_EXTENT and w <= ROW_MAX_EXTENT and sa == case.K and sx % 8 == 0 and
                sx * 2 <= ROW_MAX_BYTES and sx >= case.anchors * case.K and sy % 8 == 0 and sn % 8 == 0 and
                (case.offset * case.esize) % 16 == 0):
            return False
    return True


def candidate_masks(case: Case):
    """Per image (sure, ambiguous) masks of the reference."""
    ref = reference(case)
    return [membership(ref.scores[i], case.thr, score_band(case, ref.scores[i])) for i in range(case.n_images)]


def reference_candidates(case: Case, i: int):
    """Image i's reference candidates in row-major (anchor, class) order: fp32 boxes, scores and labels."""
    ref = reference(case)
    sure, amb = candidate_masks(case)[i]
    inds, labels = np.nonzero(sure | amb)
    return ref.boxes[i][inds].astype(np.float32), ref.scores[i][inds, labels].astype(np.float32), labels


def nms_branches(count: int, keep: np.ndarray, order_pos: np.ndarray, case: Case, boxes: np.ndarray) -> set:
    """The NMS kernel's branches for one image with `count` candidates whose full keep list (before max_det) is
    `keep`, `order_pos[j]` being candidate j's position in the sorted order."""
    p = set()
    if count == 0:
        return {"nms empty image"}
    p.add("sort bitonic R=4" if count <= 4 * NMS_THREADS else "sort bitonic R=8" if count <= SMALL_SORT else "sort radix")
    trick = count * 4 <= 4000 if case.semantics == R.TV_AUTO else case.semantics == R.OFFSET_TRICK
    if trick:
        p.add("nms trick")
        if boxes.size and boxes.min() < 0:
            p.add("nms trick, negative coordinates")
    else:
        p.add("nms per-class labmask" if case.nc <= MAX_LABEL_MASKS else "nms per-class no labmask")
    stop = len(keep) > case.max_det
    last = order_pos[keep[case.max_det - 1]] if stop else count - 1
    if last // SWEEP > 0:
        p.add("sweep multi-round")
    if stop:
        p.add("sweep max_det stop")
    return p


@functools.lru_cache(maxsize=None)
def postprocess_paths(case: Case) -> frozenset:
    """Names of the decode kernel instance, row-kernel branches, selection edges and NMS branches this case reaches."""
    p = set()
    rows = uses_rows(case)
    p.add(f"{'rows' if rows else 'candidates'} {case.dtype}")
    wide = any(w > ROW_MAX_EXTENT for _, w in case.levels)
    tall = any(h > ROW_MAX_EXTENT for h, _ in case.levels)
    if case.layout == "nhwc" and case.dtype != "f32" and not rows:
        if wide:
            p.add("nhwc W >= 1024 -> candidates")
        if tall:
            p.add("nhwc H >= 1024 -> candidates")
        if case.pitch * 2 > ROW_MAX_BYTES:
            p.add("nhwc row > 512 B -> candidates")
        if (case.offset * case.esize) % 16:
            p.add("nhwc misaligned base -> candidates")
    masks = candidate_masks(case)
    ref = reference(case)
    if rows:
        P = sum(h * w for h, w in case.levels)
        pix_start = np.cumsum([0] + [h * w for h, w in case.levels])
        for r0 in range(0, P, ROW_PIXELS):
            r1 = r0 + ROW_PIXELS - 1
            lv0 = int(np.searchsorted(pix_start, r0, "right")) - 1
            lv1 = int(np.searchsorted(pix_start, min(r1, P - 1), "right")) - 1
            if r1 >= P:
                p.add("rows partial last warp")
            if lv0 != lv1:
                p.add("rows warp straddles a level border")
            p.add("rows dense copy" if r1 < P and lv0 == lv1 and case.pitch * 2 == ROW_MAX_BYTES else "rows per-row copy")
        for sure, amb in masks:
            per_pixel = np.bincount(ref.pixel, weights=(sure | amb).sum(1), minlength=P)
            blocks = np.add.reduceat(per_pixel, np.arange(0, P, ROW_PIXELS * ROW_WARPS))
            if blocks.max() > ROW_LIST:
                p.add("rows list overflow")
        if case.thr == 0:
            p.add("rows threshold 0")
        p.add(f"rows {case.anchors} anchor" + ("s" if case.anchors > 1 else ""))
        if any(w == ROW_MAX_EXTENT for _, w in case.levels):
            p.add("rows W 1023")
    counts = [int((s | a).sum()) for s, a in masks]
    over = [c > case.cap for c in counts]
    if any(over):
        p.add("arena overflow in one image of a batch" if not all(over) else "arena overflow in every image")
    if case.max_det == 1:
        p.add("max_det 1")
    if case.max_det == 4096:
        p.add("max_det 4096")
    if case.rescale:
        p.add("rescale")
    for i, c in enumerate(counts):
        b, s, l = reference_candidates(case, i)
        keep = R.batched_nms(b, s, l, case.iou, case.semantics)
        order = np.lexsort((np.arange(c), -s.astype(np.float64)))
        pos = np.empty(c, dtype=np.int64)
        pos[order] = np.arange(c)
        p |= nms_branches(c, keep, pos, case, b)
        if case.max_det == 4096 and len(keep) >= 4096:
            p.add("max_det 4096 reached")
    if counts and max(counts) > 0:
        p.add("nms explicit")
    return frozenset(p)


# ---- the table ----------------------------------------------------------------------------------------------------------
def _cases() -> List[Case]:
    out = []
    seed = 0

    def add(**kw):
        nonlocal seed
        seed += 1
        out.append(Case(seed=seed, **kw))

    three = ((16, 24), (8, 12), (4, 6))           # 504 pixels: a warp straddles each level border, a partial last warp
    # ---- the row kernel: dtypes, anchors, pitch ----
    for dt in ("f16", "bf16"):
        add(name=f"rows {dt} 3 levels nc80", levels=three, dtype=dt)
        add(name=f"rows {dt} 1 anchor nc3 pitch 16", levels=((20, 20), (10, 10)), dtype=dt, anchors=1, nc=3, pitch=16,
            obj_shift=0.0)
        add(name=f"rows {dt} 2 anchors nc91 pitch 192", levels=((12, 40), (6, 20)), dtype=dt, anchors=2, nc=91,
            pitch=192)
        add(name=f"rows {dt} 4 anchors nc59 4 levels", levels=((16, 24), (8, 12), (4, 6), (2, 3)), dtype=dt,
            anchors=4, nc=59, obj_shift=-1.0)
    add(name="rows f16 dense 64x64 one level", levels=((64, 64),), nc=80, obj_shift=-3.0, thr=0.3)
    # threshold 0 turns the raw-logit pre-test off: every (anchor, class) pair is a candidate
    add(name="rows f16 threshold 0", levels=((8, 8), (4, 4)), nc=3, pitch=32, thr=0.0, n_images=1)
    add(name="rows bf16 threshold 0 nc80", levels=((6, 8),), dtype="bf16", thr=0.0, n_images=1, semantics=R.EXACT_PER_CLASS)
    # val.py's conf_thres = 0.001: more than 512 candidates in a 128-pixel block -> straight to the arena
    add(name="rows f16 thr 0.001 list overflow", levels=((16, 16), (8, 8)), thr=0.001, obj_shift=0.0, cls_shift=0.0,
        n_images=1, max_det=1000, cap=1 << 17)
    add(name="rows bf16 thr 0.001 list overflow max_det 4096", levels=((20, 20), (10, 10)), dtype="bf16", thr=0.001,
        obj_shift=1.0, cls_shift=0.0, spread=2.0, n_images=1, max_det=4096, cap=1 << 17)
    # the widest level the row kernel takes, and the first it must not (px / py hold 10 bits)
    add(name="rows f16 W 1023", levels=((2, 1023), (1, 512)), anchors=3, nc=3, pitch=24, n_images=1)
    add(name="nhwc f16 W 1030 -> candidates", levels=((2, 1030), (1, 515)), anchors=3, nc=3, pitch=24, n_images=1)
    add(name="nhwc bf16 H 1100 -> candidates", levels=((1100, 2),), dtype="bf16", anchors=2, nc=3, pitch=16,
        n_images=2)
    # ---- NHWC heads the row kernel does not take ----
    add(name="nhwc f16 nc91 A3 576 B row -> candidates", levels=three, nc=91, pitch=288)
    add(name="nhwc bf16 nc80 A4 688 B row -> candidates", levels=((16, 24), (8, 12)), dtype="bf16", anchors=4,
        pitch=344)
    add(name="nhwc f16 misaligned base -> candidates", levels=three, offset=4)
    add(name="nhwc bf16 misaligned base -> candidates", levels=((10, 12), (5, 6)), dtype="bf16", anchors=2, nc=20,
        pitch=56, offset=1)
    # ---- the per-anchor kernel on the reference layout ----
    for dt in ("f32", "f16", "bf16"):
        add(name=f"nahwk {dt} 3 levels", levels=three, layout="nahwk", dtype=dt)
    add(name="nahwk f32 4 anchors nc300 per-class no labmask", levels=((16, 16), (8, 8)), layout="nahwk", dtype="f32",
        anchors=4, nc=300, obj_shift=-2.0, cls_shift=-4.0, thr=0.1)
    add(name="nahwk bf16 nc300 per-class no labmask", levels=((12, 12),), layout="nahwk", dtype="bf16", nc=300,
        obj_shift=-1.0, cls_shift=-4.0, thr=0.1, semantics=R.EXACT_PER_CLASS)
    add(name="nahwk f32 1 class", levels=three, layout="nahwk", dtype="f32", anchors=1, nc=1, obj_shift=0.0)
    # ---- NMS: sort sizes, semantics, sweep, max_det, rescale ----
    add(name="nms f16 bitonic R=8", levels=((20, 20), (10, 10)), obj_shift=-3.0, n_images=1)
    add(name="nms f16 radix sort per-class", levels=((24, 24), (12, 12)), obj_shift=-1.0, n_images=1,
        cap=1 << 15)
    add(name="nms bf16 trick negative coordinates", levels=((4, 6), (2, 3)), dtype="bf16", anchors=4, nc=20,
        pitch=112, obj_shift=0.0, thr=0.1, semantics=R.OFFSET_TRICK)
    add(name="nms f16 forced trick multi-round", levels=((16, 24), (8, 12)), nc=20, pitch=80, obj_shift=0.0,
        thr=0.1, semantics=R.OFFSET_TRICK, n_images=1)
    add(name="nms f16 max_det 1", levels=three, max_det=1, obj_shift=-1.0)
    add(name="nms f32 max_det 1000 early stop", levels=((20, 20), (10, 10)), layout="nahwk", dtype="f32",
        obj_shift=-1.0, thr=0.1, max_det=1000, n_images=1, cap=1 << 16)
    add(name="nms f16 multi-round sweep max_det 4096", levels=((16, 24), (8, 12)), nc=3, pitch=24, obj_shift=0.0,
        max_det=4096, n_images=1)
    add(name="nms f16 rescale", levels=three, rescale=True, obj_shift=-1.0)
    add(name="nms bf16 rescale per-class", levels=((20, 20), (10, 10)), dtype="bf16", rescale=True, n_images=3)
    add(name="nms f32 rescale trick", levels=three, layout="nahwk", dtype="f32", rescale=True, obj_shift=-2.5,
        semantics=R.OFFSET_TRICK)
    # ---- one image overflows its share of the arena, the other does not ----
    add(name="arena overflow f16 image 0", levels=((16, 24), (8, 12)), image_shift=(3.0, -3.0), thr=0.1, cap=2048)
    add(name="arena overflow f32 image 1 of 3", levels=((12, 12),), layout="nahwk", dtype="f32",
        image_shift=(-2.0, 3.0, -4.0), thr=0.1, cap=1000, n_images=3)
    return out


CASES = _cases()


# ---- the fused decode epilogue ------------------------------------------------------------------------------------------
@dataclasses.dataclass(frozen=True)
class FusedCase:
    name: str
    levels: Tuple[Tuple[int, int], ...]      # (H, W) of each head level: one 1x1 convolution per level
    anchors: int
    nc: int
    dtype: str = "f16"
    n_images: int = 2
    Cin: int = 64
    obj_shift: float = -2.0
    cls_shift: float = -1.0
    thr: float = 0.25
    iou: float = 0.45
    max_det: int = 300
    seed: int = 0

    @property
    def width(self) -> int:
        """Decoded columns: A * (nc + 5)."""
        return self.anchors * (self.nc + 5)

    @property
    def Cout(self) -> int:
        """The head convolution's output channels: the width padded to 16, as engine's head lowering does."""
        return (self.width + 15) // 16 * 16

    @property
    def anchors_px(self) -> List[List[float]]:
        return [[float(v) for v in ANCHORS4[i][:2 * self.anchors]] for i in range(len(self.levels))]

    @property
    def strides(self) -> List[int]:
        return STRIDES[:len(self.levels)]


def fused_conv_case(fc: FusedCase, level: int):
    """The conv_cases.Case of level `level`'s head convolution (1x1, bias, no activation)."""
    import conv_cases as CC
    h, w = fc.levels[level]
    return CC.Case(f"{fc.name} level {level}", fc.n_images, h, w, fc.Cin, fc.Cout, dtype=DTYPES[fc.dtype], act=CC.NONE,
                   seed=fc.seed * 10 + level)


def fused_desc(fc: FusedCase, level: int, ptr, decode: "_C.HeadDecode"):
    """OpDesc of level `level`'s head convolution with the decode epilogue."""
    import conv_cases as CC
    d, _ = CC.build_desc(fused_conv_case(fc, level), ptr)
    d.decode = ctypes.addressof(decode)
    return d


def fake_head_decode(fc: FusedCase) -> "_C.HeadDecode":
    hd = _C.HeadDecode()
    hd.n_anchors, hd.n_classes = fc.anchors, fc.nc
    hd.keys = hd.boxes = hd.img_count = hd.img_maxc = 0x7F00_0000_0000
    return hd


def fused_paths(fc: FusedCase) -> set:
    p = {f"fused {fc.dtype}", f"fused width {fc.width}"}
    if fc.anchors == 4:
        p.add("fused 4 anchors (a == 3)")
    if len(fc.levels) > 1:
        p.add("fused two levels in one arena")
    if any((fc.n_images * h * w) % 128 for h, w in fc.levels):
        p.add("fused ragged M")
    return p


def _fused_cases() -> List[FusedCase]:
    out = []
    seed = 0

    def add(**kw):
        nonlocal seed
        seed += 1
        out.append(FusedCase(seed=seed, **kw))

    for dt in ("f16", "bf16"):
        add(name=f"fused {dt} width 255 two levels ragged", levels=((20, 20), (10, 10)), anchors=3, nc=80, dtype=dt)
        add(name=f"fused {dt} width 256 4x64", levels=((16, 16),), anchors=4, nc=59, dtype=dt, n_images=3,
            obj_shift=-1.0)
    add(name="fused f16 width 129 3x43 ragged", levels=((13, 11),), anchors=3, nc=38, Cin=32, obj_shift=-1.0)
    add(name="fused bf16 width 192 4x48 ragged", levels=((9, 14), (5, 7)), anchors=4, nc=43, Cin=96, dtype="bf16")
    return out


FUSED_CASES = _fused_cases()
