"""Baseline JPEG decoding on the GPU, bit-identical to `torchvision.io.decode_jpeg(data, mode=ImageReadMode.RGB)`.

The decoder (csrc/jpeg_decode.cu) takes SOF0/SOF1 8-bit Huffman files with one interleaved scan, gray or YCbCr,
4:4:4 / 4:2:2 / 4:2:0, with or without restart intervals: what cameras and most encoders write.  `jpeg_info` says
whether a file is in that subset and, if not, why; `decode_jpeg` raises on files outside it rather than falling
back to the CPU.
"""
from typing import List, Union

import torch
from torch import Tensor

from . import _C

__all__ = ["decode_jpeg", "jpeg_info"]

_STATUS_NAMES = {
    _C.YB_JPEG_ST_HUFFMAN: "invalid Huffman code",
    _C.YB_JPEG_ST_COEF: "coefficient index past 63",
    _C.YB_JPEG_ST_TRUNCATED: "entropy data ends early, or an interval holds the wrong number of MCUs",
    _C.YB_JPEG_ST_RESTART: "restart marker out of sequence",
    _C.YB_JPEG_ST_RANGE: "IDCT values outside the range the device reproduces exactly",
}


def _as_bytes(data) -> bytes:
    if isinstance(data, Tensor):
        if data.dtype != torch.uint8 or data.dim() != 1:
            raise ValueError(f"expected a 1-D uint8 tensor, got {data.dtype} {tuple(data.shape)}")
        return data.cpu().numpy().tobytes()
    return bytes(data)


def jpeg_info(data: Union[Tensor, bytes]) -> dict:
    """Header facts of one file (a 1-D uint8 tensor or bytes): `supported`, `reason`, `width`, `height`,
    `components`, `sampling` [(h, v) per component], `restart_interval`, and the entropy-coded segment's byte
    range `scan`.  Host only."""
    info = _C.jpeg_parse(_as_bytes(data))
    out = {"supported": bool(info.supported), "reason": info.reason.decode()}
    if info.supported:
        n = int(info.ncomp)
        out.update(width=int(info.width), height=int(info.height), components=n,
                   sampling=[(int(info.h_samp[c]), int(info.v_samp[c])) for c in range(n)],
                   restart_interval=int(info.restart_interval), scan=(int(info.scan_begin), int(info.scan_end)))
    return out


def status_text(code: int) -> str:
    return ", ".join(v for k, v in _STATUS_NAMES.items() if code & k) or "ok"


def decode_jpeg(data: Union[Tensor, List[Tensor]], device: Union[str, torch.device] = "cuda"):
    """Decodes one JPEG (a 1-D uint8 tensor of the file's bytes) or a list of them on `device` in one batch.
    Returns `[3, H, W]` uint8 CUDA tensors, CHW views of HWC memory like `torchvision.io.read_image`, with the bytes
    torchvision's CPU decoder gives in RGB mode.  Raises ValueError naming the reason for a file outside the
    supported subset and RuntimeError when a file's entropy-coded data does not decode cleanly (that check reads
    the per-image status back, so this call synchronises)."""
    single = isinstance(data, Tensor)
    items = [data] if single else list(data)
    if not items:
        return []
    device = torch.device(device)
    if device.type != "cuda":
        raise _C.NativeLibraryError("decode_jpeg runs on a CUDA device only")
    blobs, infos = [], []
    for i, d in enumerate(items):
        b = _as_bytes(d)
        info = _C.jpeg_parse(b)
        if not info.supported:
            raise ValueError(f"decode_jpeg: image {i} is outside the device decoder's subset: {info.reason.decode()}")
        blobs.append(b)
        infos.append(info)
    images, status = _C.jpeg_decode(blobs, infos, device)
    bad = [(i, int(s)) for i, s in enumerate(status.cpu().tolist()) if s]
    if bad:
        raise RuntimeError("decode_jpeg: corrupt entropy-coded data: "
                           + "; ".join(f"image {i}: {status_text(s)}" for i, s in bad))
    return images[0] if single else images
