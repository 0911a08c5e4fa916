"""ctypes binding of libyolort_b200.so (the C ABI declared in include/yolort_b200.h).

PyTorch is used here only as the owner of device memory and streams: every wrapper hands raw
`data_ptr()`s and the current CUDA stream to the native library.  There is no fallback: if the
library is missing, or a wrapper is asked to run without a CUDA device, it raises.
"""
import ctypes
import os
from typing import Dict, List, Optional, Sequence, Tuple

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
# YB_LIB_PATH: A/B timing of alternative builds of the same ABI (scripts/ab_step.py); never set in product use
LIB_PATH = os.environ.get("YB_LIB_PATH") or os.path.join(_HERE, "libyolort_b200.so")

YB_U8, YB_F16, YB_BF16, YB_F32 = 0, 1, 2, 3
YB_LAYOUT_NCHW, YB_LAYOUT_S2D16 = 0, 1
YB_OP_CONV, YB_OP_SPP_POOL, YB_OP_UPSAMPLE2X = 0, 1, 2
YB_ACT_NONE, YB_ACT_SILU, YB_ACT_HARDSWISH, YB_ACT_LEAKY01 = 0, 1, 2, 3
YB_MAX_LEVELS, YB_MAX_ANCHORS = 4, 4
NMS_TV_AUTO, NMS_EXACT_PER_CLASS, NMS_OFFSET_TRICK = 0, 1, 2

# every symbol include/yolort_b200.h declares (tests check that the built library exports all of them)
EXPORTED_SYMBOLS = (
    "yb_last_error",
    "yb_abi_version",
    "yb_letterbox_geometry",
    "yb_letterbox",
    "yb_letterbox_strided",
    "yb_scale_coords_params",
    "yb_conv_chain_supported",
    "yb_conv_config",
    "yb_plan_create",
    "yb_plan_run",
    "yb_plan_run_range",
    "yb_plan_num_launches",
    "yb_plan_destroy",
    "yb_decode_nms_workspace_bytes",
    "yb_decode_nms_debug_offset",
    "yb_decode_nms",
    "yb_decode_dense",
    "yb_nms_layout",
    "yb_nms_begin",
    "yb_nms_finish",
    "yb_decode_candidates",
    "yb_batched_nms_workspace_bytes",
    "yb_batched_nms",
)


class LetterboxGeom(ctypes.Structure):
    _fields_ = [
        ("src_h", ctypes.c_int32), ("src_w", ctypes.c_int32),
        ("new_h", ctypes.c_int32), ("new_w", ctypes.c_int32),
        ("top", ctypes.c_int32), ("left", ctypes.c_int32),
        ("ratio_h", ctypes.c_float), ("ratio_w", ctypes.c_float),
    ]


class OpDesc(ctypes.Structure):
    _fields_ = [
        ("kind", ctypes.c_int32), ("dtype", ctypes.c_int32),
        ("N", ctypes.c_int32), ("H", ctypes.c_int32), ("W", ctypes.c_int32),
        ("Cin", ctypes.c_int32), ("in_cstride", ctypes.c_int32),
        ("in_", ctypes.c_void_p),
        ("Ho", ctypes.c_int32), ("Wo", ctypes.c_int32),
        ("Cout", ctypes.c_int32), ("out_cstride", ctypes.c_int32),
        ("out", ctypes.c_void_p),
        ("ksize", ctypes.c_int32), ("stride", ctypes.c_int32), ("pad", ctypes.c_int32),
        ("act", ctypes.c_int32),
        ("weight", ctypes.c_void_p),
        ("Cin_pad", ctypes.c_int32), ("Cout_pad", ctypes.c_int32),
        ("bias", ctypes.c_void_p),
        ("residual", ctypes.c_void_p),
        ("res_cstride", ctypes.c_int32), ("reserved", ctypes.c_int32),
        ("decode", ctypes.c_void_p),
        ("chain", ctypes.c_void_p),
    ]


class ConvChain(ctypes.Structure):
    """yb_conv_chain: the pointwise tail fused onto a convolution (include/yolort_b200.h)."""
    _fields_ = [
        ("weight", ctypes.c_void_p), ("bias", ctypes.c_void_p),
        ("Cout", ctypes.c_int32), ("Cout_pad", ctypes.c_int32), ("K_pad", ctypes.c_int32),
        ("act", ctypes.c_int32),
        ("out", ctypes.c_void_p), ("out_cstride", ctypes.c_int32),
        ("own_C", ctypes.c_int32),
        ("extra", ctypes.c_void_p), ("extra_C", ctypes.c_int32), ("extra_cstride", ctypes.c_int32),
        ("store_first", ctypes.c_int32),
    ]


class HeadDecode(ctypes.Structure):
    _fields_ = [
        ("n_anchors", ctypes.c_int32), ("n_classes", ctypes.c_int32),
        ("level_start", ctypes.c_int32), ("anchors_per_image", ctypes.c_int32),
        ("stride_px", ctypes.c_float), ("anchors_px", ctypes.c_float * 8),
        ("score_thresh", ctypes.c_float),
        ("cap_per_image", ctypes.c_int64),
        ("keys", ctypes.c_void_p), ("boxes", ctypes.c_void_p),
        ("img_count", ctypes.c_void_p), ("img_maxc", ctypes.c_void_p),
    ]


class NmsLayout(ctypes.Structure):
    _fields_ = [
        ("keys", ctypes.c_void_p), ("boxes", ctypes.c_void_p),
        ("img_count", ctypes.c_void_p), ("img_maxc", ctypes.c_void_p),
        ("cap_per_image", ctypes.c_int64), ("anchors_per_image", ctypes.c_int32),
        ("level_start", ctypes.c_int32 * YB_MAX_LEVELS),
    ]


class HeadLevel(ctypes.Structure):
    _fields_ = [
        ("logits", ctypes.c_void_p), ("dtype", ctypes.c_int32),
        ("H", ctypes.c_int32), ("W", ctypes.c_int32),
        ("stride_n", ctypes.c_int64), ("stride_a", ctypes.c_int64),
        ("stride_y", ctypes.c_int64), ("stride_x", ctypes.c_int64),
        ("stride_px", ctypes.c_float),
        ("anchors_px", ctypes.c_float * (2 * YB_MAX_ANCHORS)),
    ]


class NmsParams(ctypes.Structure):
    _fields_ = [
        ("n_images", ctypes.c_int32), ("n_levels", ctypes.c_int32),
        ("n_anchors", ctypes.c_int32), ("n_classes", ctypes.c_int32),
        ("score_thresh", ctypes.c_float), ("iou_thresh", ctypes.c_float),
        ("max_det", ctypes.c_int32), ("semantics", ctypes.c_int32),
        ("max_candidates", ctypes.c_int64),
    ]


_lib = None


class NativeLibraryError(RuntimeError):
    pass


def lib() -> ctypes.CDLL:
    """Load (once) the native library; raise loudly when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise NativeLibraryError(
            f"{LIB_PATH} is missing. Build it with `python __graft_entry__.py` (nvcc, sm_90a). "
            "yolort_b200 has no PyTorch/CPU fallback path."
        )
    L = ctypes.CDLL(LIB_PATH)
    L.yb_last_error.restype = ctypes.c_char_p
    L.yb_abi_version.restype = ctypes.c_int
    L.yb_letterbox_geometry.argtypes = [
        ctypes.c_int, ctypes.POINTER(ctypes.c_int32), ctypes.c_float, ctypes.c_float, ctypes.c_int,
        ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(LetterboxGeom), ctypes.POINTER(ctypes.c_int32)]
    L.yb_letterbox.argtypes = [
        ctypes.c_int, ctypes.POINTER(ctypes.c_void_p), ctypes.c_int, ctypes.POINTER(LetterboxGeom),
        ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int,
        ctypes.c_int, ctypes.c_void_p]
    L.yb_letterbox_strided.argtypes = [
        ctypes.c_int, ctypes.POINTER(ctypes.c_void_p), ctypes.c_int, ctypes.c_int, ctypes.POINTER(LetterboxGeom),
        ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int,
        ctypes.c_int, ctypes.c_void_p]
    L.yb_scale_coords_params.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                         ctypes.POINTER(ctypes.c_float)]
    L.yb_plan_create.argtypes = [ctypes.POINTER(OpDesc), ctypes.c_int, ctypes.POINTER(ctypes.c_void_p)]
    L.yb_conv_chain_supported.argtypes = [ctypes.POINTER(OpDesc)]
    L.yb_conv_config.argtypes = [ctypes.POINTER(OpDesc), ctypes.POINTER(ctypes.c_int32)]
    L.yb_plan_run.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
    L.yb_plan_run_range.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    L.yb_plan_num_launches.argtypes = [ctypes.c_void_p]
    L.yb_plan_destroy.argtypes = [ctypes.c_void_p]
    L.yb_decode_nms_workspace_bytes.restype = ctypes.c_size_t
    L.yb_decode_nms_workspace_bytes.argtypes = [ctypes.POINTER(NmsParams), ctypes.POINTER(HeadLevel)]
    L.yb_decode_nms_debug_offset.restype = ctypes.c_size_t
    L.yb_decode_nms_debug_offset.argtypes = [ctypes.POINTER(NmsParams), ctypes.POINTER(HeadLevel)]
    L.yb_decode_nms.argtypes = [
        ctypes.POINTER(NmsParams), ctypes.POINTER(HeadLevel), ctypes.c_void_p, ctypes.c_void_p,
        ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
        ctypes.c_size_t, ctypes.c_void_p]
    L.yb_decode_dense.argtypes = [ctypes.POINTER(NmsParams), ctypes.POINTER(HeadLevel), ctypes.c_void_p,
                                  ctypes.c_void_p, ctypes.c_void_p]
    L.yb_nms_layout.argtypes = [ctypes.POINTER(NmsParams), ctypes.POINTER(HeadLevel), ctypes.c_void_p, ctypes.c_size_t,
                                ctypes.POINTER(NmsLayout)]
    L.yb_nms_begin.argtypes = [ctypes.POINTER(NmsParams), ctypes.POINTER(HeadLevel), ctypes.c_void_p, ctypes.c_void_p,
                               ctypes.c_size_t, ctypes.c_void_p]
    L.yb_nms_finish.argtypes = [ctypes.POINTER(NmsParams), ctypes.POINTER(HeadLevel), ctypes.c_void_p, ctypes.c_void_p,
                                ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                ctypes.c_size_t, ctypes.c_void_p]
    L.yb_decode_candidates.argtypes = [ctypes.POINTER(NmsParams), ctypes.POINTER(HeadLevel), ctypes.c_void_p, ctypes.c_size_t,
                                       ctypes.c_void_p]
    L.yb_batched_nms_workspace_bytes.restype = ctypes.c_size_t
    L.yb_batched_nms_workspace_bytes.argtypes = [ctypes.c_int64]
    L.yb_batched_nms.argtypes = [
        ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_float, ctypes.c_int,
        ctypes.c_int32, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
    _lib = L
    return L


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = lib().yb_last_error().decode("utf-8", "replace")
        raise NativeLibraryError(f"{what} failed (status {rc}): {msg}")


def dtype_code(dt: torch.dtype) -> int:
    try:
        return {torch.uint8: YB_U8, torch.float16: YB_F16, torch.bfloat16: YB_BF16, torch.float32: YB_F32}[dt]
    except KeyError:
        raise NativeLibraryError(f"unsupported tensor dtype {dt}") from None


def current_stream_ptr(device: torch.device) -> int:
    return torch.cuda.current_stream(device).cuda_stream


class _NoGuard:
    def __enter__(self):
        return None

    def __exit__(self, *a):
        return False


_NO_GUARD = _NoGuard()


def device_guard(device: torch.device):
    """Context manager that makes `device` the current CUDA device for the native launches inside it (the kernels are
    launched on `device`'s current stream, which must belong to the current device: the reference works on any
    device, and so does this path).  Free when `device` already is current."""
    idx = device.index if device.index is not None else torch.cuda.current_device()
    if torch.cuda.current_device() == idx:
        return _NO_GUARD
    return torch.cuda.device(idx)


def require_cuda(t: torch.Tensor, what: str) -> None:
    if not t.is_cuda:
        raise NativeLibraryError(
            f"{what}: tensor lives on {t.device}; the yolort_b200 path runs on sm_90a only (no CPU fallback)")


# ---------------------------------------------------------------------------------------------------
# letterbox
# ---------------------------------------------------------------------------------------------------
def letterbox_geometry(sizes: Sequence[Tuple[int, int]], min_size: float, max_size: float,
                       size_divisible: int = 32, fixed_shape: Optional[Tuple[int, int]] = None):
    """Host-only geometry of the letterbox (transform.py:53-97, :297-330). Returns (geoms, (Hb, Wb))."""
    n = len(sizes)
    hw = (ctypes.c_int32 * (2 * n))(*[int(v) for s in sizes for v in s])
    geoms = (LetterboxGeom * n)()
    bhw = (ctypes.c_int32 * 2)()
    fs = None
    if fixed_shape is not None:
        fs = (ctypes.c_int32 * 2)(int(fixed_shape[0]), int(fixed_shape[1]))
    check(lib().yb_letterbox_geometry(n, hw, float(min_size), float(max_size), int(size_divisible), fs, geoms, bhw),
          "yb_letterbox_geometry")
    return geoms, (int(bhw[0]), int(bhw[1]))


def scale_coords_params(Hb: int, Wb: int, h: int, w: int) -> Tuple[float, float, float]:
    out = (ctypes.c_float * 3)()
    check(lib().yb_scale_coords_params(int(Hb), int(Wb), int(h), int(w), out), "yb_scale_coords_params")
    return float(out[0]), float(out[1]), float(out[2])


_u8_lut: Dict[torch.device, torch.Tensor] = {}


def u8_lut(device: torch.device) -> torch.Tensor:
    """[256] fp32 table of torch's own `uint8 / 255.0` (the default loader's normalisation,
    yolort/models/yolov5.py:228), so uint8 inputs reproduce it bit for bit."""
    t = _u8_lut.get(device)
    if t is None:
        t = (torch.arange(256, dtype=torch.uint8) / 255.0).to(torch.float32).to(device)
        _u8_lut[device] = t
    return t


YB_SRC_CHW, YB_SRC_HWC = 0, 1


def _is_hwc_view(im: torch.Tensor) -> bool:
    _, h, w = im.shape
    return tuple(im.stride()) == (1, 3 * w, 3) and (h > 1 or w > 1)


def letterbox(images: List[torch.Tensor], geoms, Hb: int, Wb: int, fill: float, out: torch.Tensor,
              layout: int) -> torch.Tensor:
    n = len(images)
    dev = out.device
    require_cuda(out, "letterbox")
    src_dtype = images[0].dtype
    ptrs = (ctypes.c_void_p * n)()
    keep = []
    for im in images:
        require_cuda(im, "letterbox")
        if im.dtype != src_dtype:
            raise NativeLibraryError("letterbox: all images of a batch must share a dtype")
        if im.dim() != 3 or im.shape[0] != 3:
            raise ValueError(f"images is expected to be a list of 3d tensors of shape [C, H, W], but got '{im.shape}'.")
    # [3,H,W] views of interleaved HWC memory (decoded image files) are read in place; anything else goes planar
    hwc = all(_is_hwc_view(im) for im in images)
    for i, im in enumerate(images):
        if not hwc:
            im = im.contiguous()
        keep.append(im)
        ptrs[i] = im.data_ptr()
    lut = u8_lut(dev) if src_dtype == torch.uint8 else None
    with device_guard(dev):
        check(lib().yb_letterbox_strided(n, ptrs, dtype_code(src_dtype), YB_SRC_HWC if hwc else YB_SRC_CHW, geoms,
                                         int(Hb), int(Wb), float(fill), lut.data_ptr() if lut is not None else None,
                                         out.data_ptr(), dtype_code(out.dtype), int(layout), current_stream_ptr(dev)),
              "yb_letterbox")
    # the kernel reads the sources asynchronously on this stream: one record per distinct storage (the images of a
    # packed batch are views of one buffer)
    stream = torch.cuda.current_stream(dev)
    seen = set()
    for im in keep:
        key = im.untyped_storage().data_ptr()
        if key not in seen:
            seen.add(key)
            im.record_stream(stream)
    return out


# ---------------------------------------------------------------------------------------------------
# execution plan
# ---------------------------------------------------------------------------------------------------
def conv_chain_supported(op: "OpDesc") -> bool:
    """Whether the native library can run `op` (with op.chain set) as one fused launch (pure host logic)."""
    return bool(lib().yb_conv_chain_supported(ctypes.byref(op)))


def conv_config(op: "OpDesc") -> dict:
    """How the library would launch this convolution (host-only): kernel, tiling, residency, shared memory."""
    info = (ctypes.c_int32 * 12)()
    check(lib().yb_conv_config(ctypes.byref(op), info), "yb_conv_config")
    keys = ("patch_kernel", "block_n", "n_tiles", "weights_resident", "tiles_per_pass", "slots", "ring", "store_cols",
            "store_bufs", "smem_bytes", "grid", "chained")
    cfg = dict(zip(keys, [int(v) for v in info]))
    if not cfg["patch_kernel"]:     # slot 8 of the 1x1 / im2col kernel: consumer warpgroups (sharing two staging buffers)
        cfg["epilogue_groups"] = cfg.pop("store_bufs")
    return cfg


class Plan:
    """Owns a native yb_plan handle (list of prepared launches)."""

    def __init__(self, ops: Sequence[OpDesc], device: torch.device):
        arr = (OpDesc * len(ops))(*ops)
        handle = ctypes.c_void_p()
        with torch.cuda.device(device):
            check(lib().yb_plan_create(arr, len(ops), ctypes.byref(handle)), "yb_plan_create")
        self._h = handle
        self.device = device
        self.n_ops = len(ops)

    def run(self, first: int = 0, count: Optional[int] = None) -> None:
        if count is None:
            count = self.n_ops - first
        with device_guard(self.device):
            check(lib().yb_plan_run_range(self._h, first, count, current_stream_ptr(self.device)), "yb_plan_run")

    def __del__(self):
        h = getattr(self, "_h", None)
        if h is not None and _lib is not None:
            _lib.yb_plan_destroy(h)
            self._h = None


# ---------------------------------------------------------------------------------------------------
# post-process
# ---------------------------------------------------------------------------------------------------
class _NmsArena:
    """Per-device reusable workspace; grows when the candidate count exceeds its capacity."""

    def __init__(self):
        self.ws: Optional[torch.Tensor] = None
        self.cap_per_image = 16384


_arenas: Dict[torch.device, _NmsArena] = {}


def _level_struct(t: torch.Tensor, layout: str, n_anchors: int, n_outputs: int, stride_px: float,
                  anchors: Sequence[float]) -> HeadLevel:
    lv = HeadLevel()
    lv.logits = t.data_ptr()
    lv.dtype = dtype_code(t.dtype)
    if layout == "nahwk":  # reference layout [N, A, H, W, K]
        if t.dim() != 5 or t.shape[1] != n_anchors or t.shape[4] != n_outputs or not t.is_contiguous():
            raise NativeLibraryError(f"decode_nms: expected contiguous [N,{n_anchors},H,W,{n_outputs}], got {tuple(t.shape)}")
        N, A, H, W, K = t.shape
        lv.H, lv.W = H, W
        lv.stride_n, lv.stride_a, lv.stride_y, lv.stride_x = A * H * W * K, H * W * K, W * K, K
    elif layout == "nhwc":  # plan layout [N, H, W, Cpad] with channel a*K + k
        if t.dim() != 4 or t.shape[3] < n_anchors * n_outputs or not t.is_contiguous():
            raise NativeLibraryError(f"decode_nms: expected contiguous [N,H,W,>={n_anchors * n_outputs}], got {tuple(t.shape)}")
        N, H, W, C = t.shape
        lv.H, lv.W = H, W
        lv.stride_n, lv.stride_a, lv.stride_y, lv.stride_x = H * W * C, n_outputs, W * C, C
    else:
        raise NativeLibraryError(f"unknown head layout {layout!r}")
    lv.stride_px = float(stride_px)
    for i, v in enumerate(anchors):
        lv.anchors_px[i] = float(v)
    return lv


def decode_nms_padded(head_outputs: List[torch.Tensor], layout: str, strides: Sequence[float],
                      anchors_px: Sequence[Sequence[float]], num_classes: int, score_thresh: float,
                      nms_thresh: float, detections_per_img: int, semantics: int = NMS_TV_AUTO,
                      rescale: Optional[torch.Tensor] = None, stage_hook=None):
    """Launches decode+NMS; returns padded device tensors (boxes [N,D,4], scores [N,D], labels [N,D],
    counts [N], status [4]) without synchronising -- the caller reads `counts`/`status`."""
    t0 = head_outputs[0]
    require_cuda(t0, "decode_nms")
    dev = t0.device
    n_images = int(t0.shape[0])
    n_levels = len(head_outputs)
    n_anchors = len(anchors_px[0]) // 2
    if n_levels > YB_MAX_LEVELS or n_anchors > YB_MAX_ANCHORS:
        raise NativeLibraryError("decode_nms: too many levels/anchors")
    arena = _arenas.setdefault(dev, _NmsArena())
    levels = (HeadLevel * n_levels)(*[
        _level_struct(t, layout, n_anchors, num_classes + 5, strides[i], anchors_px[i])
        for i, t in enumerate(head_outputs)])
    D = int(detections_per_img)
    boxes = torch.empty((n_images, D, 4), dtype=torch.float32, device=dev)
    scores = torch.empty((n_images, D), dtype=torch.float32, device=dev)
    labels = torch.empty((n_images, D), dtype=torch.int64, device=dev)
    counts = torch.empty((n_images,), dtype=torch.int32, device=dev)
    status = torch.empty((4,), dtype=torch.int64, device=dev)
    p = NmsParams(n_images, n_levels, n_anchors, int(num_classes), float(score_thresh), float(nms_thresh), D,
                  int(semantics), int(arena.cap_per_image) * n_images)
    need = lib().yb_decode_nms_workspace_bytes(ctypes.byref(p), levels)
    if arena.ws is None or arena.ws.numel() < need or arena.ws.device != dev:
        arena.ws = torch.empty((need,), dtype=torch.uint8, device=dev)
    with device_guard(dev):
        if stage_hook is None:
            check(lib().yb_decode_nms(ctypes.byref(p), levels, rescale.data_ptr() if rescale is not None else None,
                                      boxes.data_ptr(), scores.data_ptr(), labels.data_ptr(), counts.data_ptr(),
                                      status.data_ptr(), arena.ws.data_ptr(), arena.ws.numel(), current_stream_ptr(dev)),
                  "yb_decode_nms")
        else:   # same three steps, with a callback between them (bench.py records CUDA events per stage)
            st = current_stream_ptr(dev)
            check(lib().yb_nms_begin(ctypes.byref(p), levels, status.data_ptr(), arena.ws.data_ptr(), arena.ws.numel(), st),
                  "yb_nms_begin")
            stage_hook("begin")
            check(lib().yb_decode_candidates(ctypes.byref(p), levels, arena.ws.data_ptr(), arena.ws.numel(), st),
                  "yb_decode_candidates")
            stage_hook("decode")
            check(lib().yb_nms_finish(ctypes.byref(p), levels, rescale.data_ptr() if rescale is not None else None,
                                      boxes.data_ptr(), scores.data_ptr(), labels.data_ptr(), counts.data_ptr(),
                                      status.data_ptr(), arena.ws.data_ptr(), arena.ws.numel(), st), "yb_nms_finish")
            stage_hook("nms")
    arena.debug_offset = lib().yb_decode_nms_debug_offset(ctypes.byref(p), levels)
    return boxes, scores, labels, counts, status


def decode_dense(head_outputs: List[torch.Tensor], layout: str, strides: Sequence[float],
                 anchors_px: Sequence[Sequence[float]], num_classes: int):
    """LogitsDecoder (yolort/relay/logits_decoder.py:26-61): (boxes [N,A,4] xyxy fp32, scores [N,A,nc] fp32) for
    every anchor, no threshold and no NMS; one launch, no host synchronisation."""
    t0 = head_outputs[0]
    require_cuda(t0, "decode_dense")
    dev = t0.device
    n_images, n_levels = int(t0.shape[0]), len(head_outputs)
    n_anchors = len(anchors_px[0]) // 2
    if n_levels > YB_MAX_LEVELS or n_anchors > YB_MAX_ANCHORS:
        raise NativeLibraryError("decode_dense: too many levels/anchors")
    levels = (HeadLevel * n_levels)(*[
        _level_struct(t, layout, n_anchors, num_classes + 5, strides[i], anchors_px[i])
        for i, t in enumerate(head_outputs)])
    total = sum(n_anchors * int(lv.H) * int(lv.W) for lv in levels)
    boxes = torch.empty((n_images, total, 4), dtype=torch.float32, device=dev)
    scores = torch.empty((n_images, total, int(num_classes)), dtype=torch.float32, device=dev)
    p = NmsParams(n_images, n_levels, n_anchors, int(num_classes), 0.0, 0.0, 1, 0, 0)
    with device_guard(dev):
        check(lib().yb_decode_dense(ctypes.byref(p), levels, boxes.data_ptr(), scores.data_ptr(), current_stream_ptr(dev)),
              "yb_decode_dense")
    return boxes, scores


def nms_phase_clocks(device) -> list:
    """Debug: clock counts of the NMS kernel phases for image 0 of the last decode_nms call on `device`."""
    arena = _arenas[torch.device(device)]
    off = arena.debug_offset
    return arena.ws[off: off + 128].view(torch.int64)[4:10].cpu().tolist()


def decode_nms(head_outputs: List[torch.Tensor], layout: str, strides, anchors_px, score_thresh: float,
               nms_thresh: float, detections_per_img: int, semantics: int = NMS_TV_AUTO,
               rescale: Optional[torch.Tensor] = None, num_classes: Optional[int] = None) -> List[Dict[str, torch.Tensor]]:
    """Full post-process returning the reference's List[Dict] (keys in order scores, labels, boxes:
    yolort/models/box_head.py:427).  One device->host read of counts+status; re-runs with a larger
    arena when an image overflowed its candidate share (never truncates silently)."""
    if num_classes is None:
        t0 = head_outputs[0]
        num_classes = int(t0.shape[4]) - 5 if layout == "nahwk" else None
        if num_classes is None:
            raise NativeLibraryError("decode_nms: num_classes is required for the nhwc layout")
    dev = head_outputs[0].device
    while True:
        boxes, scores, labels, counts, status = decode_nms_padded(
            head_outputs, layout, strides, anchors_px, num_classes, score_thresh, nms_thresh,
            detections_per_img, semantics, rescale)
        host = torch.cat([counts.to(torch.int64), status]).tolist()     # one D2H + one conversion for the whole batch
        n = counts.numel()
        if host[n + 1] == 0:
            break
        arena = _arenas[dev]
        arena.cap_per_image = max(2 * arena.cap_per_image, int(host[n + 2]))
        arena.ws = None
    return [{"scores": scores[i, :host[i]], "labels": labels[i, :host[i]], "boxes": boxes[i, :host[i]]} for i in range(n)]


class FusedPost:
    """Post-processing state of a plan whose head convolutions decode in their epilogue: a fixed candidate arena
    (the heads hold raw pointers into it), the NMS parameters, and begin()/finish() around the plan run."""

    def __init__(self, n_images: int, level_hw: Sequence[Tuple[int, int]], strides: Sequence[float],
                 anchors_px: Sequence[Sequence[float]], num_classes: int, score_thresh: float, nms_thresh: float,
                 detections_per_img: int, semantics: int, device: torch.device, cap_per_image: int = 32768):
        self.device = device
        self.n_images, self.D = n_images, int(detections_per_img)
        n_levels, n_anchors = len(level_hw), len(anchors_px[0]) // 2
        self.levels = (HeadLevel * n_levels)()
        for i, (h, w) in enumerate(level_hw):
            self.levels[i].H, self.levels[i].W = int(h), int(w)
            self.levels[i].dtype = YB_F16
            self.levels[i].stride_px = float(strides[i])
            for j, v in enumerate(anchors_px[i]):
                self.levels[i].anchors_px[j] = float(v)
        self.params = NmsParams(n_images, n_levels, n_anchors, int(num_classes), float(score_thresh), float(nms_thresh),
                                self.D, int(semantics), int(cap_per_image) * n_images)
        need = lib().yb_decode_nms_workspace_bytes(ctypes.byref(self.params), self.levels)
        self.ws = torch.empty((need,), dtype=torch.uint8, device=device)
        self.layout = NmsLayout()
        check(lib().yb_nms_layout(ctypes.byref(self.params), self.levels, self.ws.data_ptr(), self.ws.numel(),
                                  ctypes.byref(self.layout)), "yb_nms_layout")
        self.head_decode = []
        for i in range(n_levels):
            hd = HeadDecode()
            hd.n_anchors, hd.n_classes = n_anchors, int(num_classes)
            hd.level_start, hd.anchors_per_image = int(self.layout.level_start[i]), int(self.layout.anchors_per_image)
            hd.stride_px = float(strides[i])
            for j, v in enumerate(anchors_px[i]):
                hd.anchors_px[j] = float(v)
            hd.score_thresh = float(score_thresh)
            hd.cap_per_image = int(self.layout.cap_per_image)
            hd.keys, hd.boxes = self.layout.keys, self.layout.boxes
            hd.img_count, hd.img_maxc = self.layout.img_count, self.layout.img_maxc
            self.head_decode.append(hd)
        self.status = torch.empty((4,), dtype=torch.int64, device=device)

    def begin(self) -> None:
        with device_guard(self.device):
            check(lib().yb_nms_begin(ctypes.byref(self.params), self.levels, self.status.data_ptr(), self.ws.data_ptr(),
                                     self.ws.numel(), current_stream_ptr(self.device)), "yb_nms_begin")

    def finish(self, rescale: Optional[torch.Tensor]):
        n, D, dev = self.n_images, self.D, self.device
        boxes = torch.empty((n, D, 4), dtype=torch.float32, device=dev)
        scores = torch.empty((n, D), dtype=torch.float32, device=dev)
        labels = torch.empty((n, D), dtype=torch.int64, device=dev)
        counts = torch.empty((n,), dtype=torch.int32, device=dev)
        with device_guard(dev):
            check(lib().yb_nms_finish(ctypes.byref(self.params), self.levels,
                                      rescale.data_ptr() if rescale is not None else None, boxes.data_ptr(),
                                      scores.data_ptr(), labels.data_ptr(), counts.data_ptr(), self.status.data_ptr(),
                                      self.ws.data_ptr(), self.ws.numel(), current_stream_ptr(dev)), "yb_nms_finish")
        return boxes, scores, labels, counts, self.status


def batched_nms(boxes: torch.Tensor, scores: torch.Tensor, labels: torch.Tensor, iou_threshold: float,
                semantics: int = NMS_TV_AUTO, max_keep: int = 4096) -> torch.Tensor:
    """torchvision.ops.batched_nms on the device (first `max_keep` survivors, score-descending)."""
    require_cuda(boxes, "batched_nms")
    dev = boxes.device
    boxes = boxes.contiguous().float()
    scores = scores.contiguous().float()
    labels = labels.contiguous().to(torch.int64)
    n = int(boxes.shape[0])
    keep = torch.empty((max_keep,), dtype=torch.int64, device=dev)
    n_keep = torch.zeros((1,), dtype=torch.int32, device=dev)
    need = lib().yb_batched_nms_workspace_bytes(n)
    ws = torch.empty((need,), dtype=torch.uint8, device=dev)
    with device_guard(dev):
        check(lib().yb_batched_nms(boxes.data_ptr(), scores.data_ptr(), labels.data_ptr(), n, float(iou_threshold),
                                   int(semantics), int(max_keep), keep.data_ptr(), n_keep.data_ptr(), ws.data_ptr(),
                                   ws.numel(), current_stream_ptr(dev)), "yb_batched_nms")
    return keep[: int(n_keep.item())]
