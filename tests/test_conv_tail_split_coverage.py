"""The split tail of the 1x1 / im2col kernel: every instance that has tail slices is reached with and without them,
the rule holds at its edges, and the reserved bit keeps the tiles whole (host logic, no GPU needed; SM-dependent sizes
follow the device's SM count, 132 without a GPU)."""
import re

import conv_cases
import conv_cases_one_group as og
import conv_cases_tail_split as ts
from conv_cases import build_desc, fake_ptr
from test_conv_one_group_coverage import _selector
from yolort_b200 import _C


def _plan(c, extra=0):
    d, _ch = build_desc(c, fake_ptr)
    d.reserved |= extra
    return _C.conv_config(d)


def split_instances() -> set:
    """(dtype, N, layout) of every 128-column instance without a decode or a tail: the ones with tail slices."""
    src = _selector()
    out = set()
    for dt in ("f16", "bf16"):
        for m in re.finditer(r"conv_wgmma_kernel<kBf16, 128, false, 0, (\d)(?:, (\d))?>", src):
            out.add((dt, 128, f"{m[1]}x{m[2] or 2}"))
    return out


def test_case_names_are_unique():
    names = [c.name for c in ts.CASES]
    assert len(names) == len(set(names))
    assert not set(names) & {c.name for c in conv_cases.CASES + og.CASES}


def test_cases_take_the_path_their_name_states():
    for c in ts.CASES:
        cfg = _plan(c)
        split = c.name.split()[1] == "split"
        block_n = 256 if c.name.split()[1] == "whole256" else 128
        assert cfg["layout"] == c.name.split()[2] and cfg["block_n"] == block_n, (c.name, cfg)
        assert cfg["tail_split"] == (2 if split else 1), (c.name, cfg)
        r = cfg["work_items"] % cfg["grid"]
        assert cfg["tail_tiles"] == (r if split else 0), (c.name, cfg)
        if split:
            assert 0 < 2 * r <= cfg["grid"] and cfg["grid"] % cfg["n_tiles"] == 0, (c.name, cfg)


def test_every_split_instance_is_reached_with_and_without_slices():
    inst = split_instances()
    assert inst == {(dt, 128, lay) for dt in ("f16", "bf16") for lay in ("1x2", "2x1")}, sorted(inst)
    reached = {}
    for c in ts.CASES + og.CASES + conv_cases.CASES:
        cfg = _plan(c)
        if not cfg["patch_kernel"] and not cfg["chained"]:
            reached.setdefault(ts.split_key(c, cfg), []).append(c.name)
    for dt, n, lay in sorted(inst):
        for split in (1, 2):
            print(f"  {(dt, n, lay, split)}: {reached.get((dt, n, lay, split), 'MISSING')}")
            assert (dt, n, lay, split) in reached


def test_streamed_and_im2col_slices_are_reached():
    paths = set()
    for c in ts.CASES:
        cfg = _plan(c)
        if cfg["tail_split"] == 2:
            paths.add("streamed" if not cfg["weights_resident"] else "resident")
            paths.add("1x1" if c.k == 1 else "im2col")
            if cfg["n_tiles"] > 1:
                paths.add("several N tiles")
            if c.Cout % 128:
                paths.add("ragged Cout")
            if c.Cout == 256 and cfg["layout"] == "1x2":
                paths.add("256 columns as two N tiles")
    assert paths == {"streamed", "resident", "1x1", "im2col", "several N tiles", "ragged Cout",
                     "256 columns as two N tiles"}, paths


def test_no_tail_split_bit_keeps_the_tiles_whole():
    for c in ts.CASES:
        cfg = _plan(c)
        whole = _plan(c, _C.YB_CONV_NO_TAIL_SPLIT)
        assert whole["tail_split"] == 1 and whole["tail_tiles"] == 0, (c.name, whole)
        if cfg["tail_split"] == 2 and c.Cout == 256 and cfg["layout"] == "1x2":   # keeps the 256-column tile
            assert (whole["block_n"], whole["n_tiles"]) == (256, 1), (c.name, whole)
            continue
        for k in ("layout", "block_n", "n_tiles", "grid", "work_items", "weights_resident", "slots", "smem_bytes"):
            assert whole[k] == cfg[k], (c.name, k)


def test_other_instances_never_split():
    for c in conv_cases.CASES + og.CASES:
        cfg = _plan(c)
        if cfg["tail_split"] > 1:
            assert not cfg["patch_kernel"] and not cfg["chained"] and cfg["block_n"] == 128, (c.name, cfg)
