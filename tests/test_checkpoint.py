"""Upstream-checkpoint loader vs the reference converter (CPU).  The synthetic upstream checkpoints (the vendored
ultralytics `Model`, pickled with classes models.yolo.* / models.common.*) and the reference converter's output on
them are stored in tests/golden/upstream_ckpt_*.npz (oracle/make_golden_checkpoint.py); tests/checkpoint_util.py
rebuilds the checkpoints without the reference tree."""
import json
import os
import sys

import numpy as np
import pytest

import checkpoint_util as cu


def _fixture(golden_dir, tag):
    return np.load(os.path.join(golden_dir, f"upstream_ckpt_{tag}.npz"))


def _checkpoint(tmp_path_factory, golden_dir, tag):
    path = str(tmp_path_factory.mktemp("ckpt") / f"yolov5{tag}_synth.pt")
    cu.rebuild_checkpoint(_fixture(golden_dir, tag), path)
    # the loader under test must not need the upstream tree on sys.path
    assert not any(k == "models" or k.startswith("models.") for k in sys.modules)
    return path


def _reference_output(golden_dir, tag):
    return json.loads(bytes(_fixture(golden_dir, tag)["converted"]).decode())


@pytest.fixture(scope="module")
def upstream_ckpt(tmp_path_factory, golden_dir):
    """A synthetic upstream yolov5n checkpoint, pickled exactly like ultralytics does."""
    return _checkpoint(tmp_path_factory, golden_dir, "n")


@pytest.fixture(scope="module")
def upstream_ckpt_p6(tmp_path_factory, golden_dir):
    return _checkpoint(tmp_path_factory, golden_dir, "n6")


def _assert_equals_reference(mine, ref):
    got = cu.describe(mine)
    assert got["num_classes"] == ref["num_classes"] == 80
    assert got["strides"] == ref["strides"]
    assert got["anchor_grids"] == ref["anchor_grids"]
    assert got["keys"] == ref["keys"]
    for k, want in ref["tensors"].items():
        assert got["tensors"][k] == want, k


def test_converted_state_dict_equals_reference_converter(upstream_ckpt, golden_dir):
    from yolort_b200.models._checkpoint import load_from_ultralytics

    mine = load_from_ultralytics(upstream_ckpt)
    assert (mine["depth_multiple"], mine["width_multiple"], mine["size"]) == (0.33, 0.25, "n")
    assert mine["strides"] == [8, 16, 32] and isinstance(mine["strides"][0], int)
    _assert_equals_reference(mine, _reference_output(golden_dir, "n"))


def test_load_from_yolov5_builds_a_model(upstream_ckpt):
    from yolort_b200.models import YOLOv5

    m = YOLOv5.load_from_yolov5(upstream_ckpt, score_thresh=0.3)
    assert m.model.post_process.score_thresh == 0.3
    assert m.model.anchor_generator.strides == [8, 16, 32]
    assert len(m.state_dict()) == 348


def test_p6_checkpoint_equals_reference_converter(upstream_ckpt_p6, golden_dir):
    """_checkpoint.py:49-58: 4 strides -> use_p6, module index maps of the 34-module upstream graph."""
    from yolort_b200.models import YOLOv5
    from yolort_b200.models._checkpoint import load_from_ultralytics

    mine = load_from_ultralytics(upstream_ckpt_p6)
    assert mine["use_p6"] is True
    assert mine["strides"] == [8, 16, 32, 64]
    _assert_equals_reference(mine, _reference_output(golden_dir, "n6"))
    m = YOLOv5.load_from_yolov5(upstream_ckpt_p6, size_divisible=64)
    assert m.model.anchor_generator.strides == [8, 16, 32, 64] and len(m.model.head.head) == 4
