"""Host side of the device JPEG decoder: yb_jpeg_parse (geometry, routing reasons, hostile headers) and the numpy
restatement of the CPU decoder (oracle/restate_jpeg.py) against torchvision and the committed digests."""
import ctypes
import json
import os
import struct
import subprocess

import numpy as np
import pytest

import jpeg_corpus as J
from oracle import restate_jpeg as RJ
from yolort_b200 import _C
from yolort_b200.io import jpeg_info

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _digests():
    with open(os.path.join(J.GOLDEN_JPEG, "digests.json")) as f:
        return json.load(f)


def test_info_struct_matches_header(tmp_path):
    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "yolort_b200.h"\n'
                   'int main(void){printf("%zu %zu %zu\\n", sizeof(yb_jpeg_info), offsetof(yb_jpeg_info, data_offset), '
                   'offsetof(yb_jpeg_info, ac_vals));return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert got == [ctypes.sizeof(_C.JpegInfo), _C.JpegInfo.data_offset.offset, _C.JpegInfo.ac_vals.offset]


@pytest.mark.parametrize("sizes", [J.SMALL_SIZES, J.LARGE_SIZES])
def test_parse_reports_geometry(sizes):
    files = J.corpus(sizes) + J.cv2_corpus(sizes if sizes == J.SMALL_SIZES else ())
    assert len(files) > 20
    for name, data, want in files:
        got = jpeg_info(data)
        assert got["supported"], (name, got["reason"])
        for k, v in want.items():
            if v is not None:
                assert got[k] == v, (name, k, got[k], v)
        assert got["scan"] == J.scan_segment(data), name


def test_parse_assets():
    bus, zidane = (jpeg_info(d) for _, d in J.assets())
    assert (bus["width"], bus["height"], bus["restart_interval"], bus["sampling"]) == (810, 1080, 51, [(2, 2), (1, 1), (1, 1)])
    assert (zidane["width"], zidane["height"], zidane["restart_interval"]) == (1280, 720, 0)
    assert zidane["sampling"] == [(2, 2), (1, 1), (1, 1)]


def _sof_offset(data: bytes) -> int:
    return data.index(b"\xff\xc0")


def test_parse_reasons():
    assert "progressive" in jpeg_info(J.progressive())["reason"]
    assert "4 components" in jpeg_info(J.cmyk())["reason"]
    base = J.pil_jpeg(J.photo(16, 24, 1), quality=80, subsampling=2)
    i = _sof_offset(base)
    twelve = bytearray(base)
    twelve[i + 4] = 12                                  # hand-built header: 12-bit sample precision
    assert "12-bit" in jpeg_info(bytes(twelve))["reason"]
    # one component per scan (a baseline multi-scan file): rewrite the SOS to carry the first component only
    s = base.index(b"\xff\xda")
    ln = base[s + 2] << 8 | base[s + 3]
    first = base[s + 5:s + 7]
    sos = b"\xff\xda" + struct.pack(">HB", 8, 1) + first + b"\x00\x3f\x00"
    multi = base[:s] + sos + base[s + 2 + ln:]
    assert "multi-scan" in jpeg_info(multi)["reason"]
    assert "not a JPEG" in jpeg_info(b"\x89PNG\r\n\x1a\n" + bytes(32))["reason"]
    assert not jpeg_info(b"")["supported"]
    adobe_rgb = base[:2] + b"\xff\xee\x00\x0eAdobe\x00\x64\x00\x00\x00\x00\x00" + base[2:]
    adobe_rgb = adobe_rgb.replace(b"JFIF\x00", b"JFIX\x00", 1)
    assert "RGB" in jpeg_info(adobe_rgb)["reason"]
    h1v2 = bytearray(base)
    h1v2[i + 11] = 0x12                                 # luma 1x2: a 4:4:0 file
    assert "sampling ratio" in jpeg_info(bytes(h1v2))["reason"]


def test_parse_survives_truncated_and_mutated_headers():
    base = J.pil_jpeg(J.photo(33, 47, 2), quality=90, subsampling=2, restart_marker_blocks=2)
    b0, _ = J.scan_segment(base)
    for k in range(0, b0 + 8):
        assert not jpeg_info(base[:k])["supported"], k
    rng = np.random.default_rng(0)
    seen = set()
    for _ in range(3000):
        m = bytearray(base)
        for _ in range(int(rng.integers(1, 4))):
            m[int(rng.integers(0, b0))] = int(rng.integers(0, 256))
        info = jpeg_info(bytes(m))
        seen.add(info["supported"])
        if info["supported"]:        # whatever the header says, the geometry it reports is self-consistent
            assert info["width"] >= 1 and info["height"] >= 1
            assert b0 - 64 <= info["scan"][0] <= info["scan"][1] <= len(m)
    assert seen == {True, False}


@pytest.mark.parametrize("source", ["pil", "cv2"])
def test_restatement_equals_torchvision(source):
    files = J.corpus() if source == "pil" else J.cv2_corpus()
    if not files:
        pytest.skip("cv2 is not installed")
    for name, data, _ in files:
        got = RJ.decode(data)
        want = J.cpu_decode(data).numpy()
        assert np.array_equal(got, want), name


def test_restatement_equals_torchvision_at_edge_sizes():
    for (h, w) in ((2, 2), (3, 3), (4, 5), (9, 7), (16, 16), (17, 33)):
        a = J.photo(h, w, h * 31 + w)
        for q in (50, 100):
            for ss in (0, 1, 2):
                data = J.pil_jpeg(a, quality=q, subsampling=ss)
                assert np.array_equal(RJ.decode(data), J.cpu_decode(data).numpy()), (h, w, q, ss)


def test_cpu_decoder_matches_committed_digests():
    dig = _digests()
    files = J.assets() + [(n, b) for n, b, _ in J.corpus(sizes=((61, 117),))]
    checked = 0
    for name, data in files:
        d = dig[name]
        if d["file"] != J.sha(data):        # a different PIL encodes different bytes: nothing to compare
            continue
        assert J.sha(J.cpu_decode(data).numpy().tobytes()) == d["rgb"], name
        checked += 1
    assert checked >= 2                     # the two committed camera files at least


def test_restatement_matches_committed_digests_on_assets():
    dig = _digests()
    for name, data in J.assets():
        assert J.sha(RJ.decode(data).tobytes()) == dig[name]["rgb"], name
