"""The case table of tests/conv_cases.py reaches every fp16/bf16 convolution kernel instance and every plan path (host
logic, no GPU needed; SM-dependent sizes follow the device's SM count, 132 without a GPU).

The instance list comes from the kernel selectors' source, so a new instance fails this test until a case reaches it.
"""
import os
import re

from conv_cases import CASES, EXCLUDED, SMS, build_desc, fake_ptr, instance_key, plan_paths
from yolort_b200 import _C

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "yolort_b200", "csrc")

REQUIRED_PATHS = {
    # 1x1 / im2col kernel
    "conv 1x1 resident", "conv 1x1 streamed",
    "conv im2col 3x3 s1 resident", "conv im2col 3x3 s1 streamed",
    "conv im2col 3x3 s2 resident", "conv im2col 3x3 s2 streamed",
    "conv several N tiles", "conv im2col k5",
    # halo-patch kernel
    "patch classic", "patch wrap", "patch stride2",
    "patch resident single N tile", "patch resident N-split", "patch streamed pairs", "patch streamed odd last pair",
    # two CTAs per SM
    "two CTAs conv", "two CTAs patch classic", "two CTAs patch wrap", "two CTAs patch stride2",
    "two CTAs at 2 x SMs tiles", "one CTA at 2 x SMs - 1 tiles",
    # chained tails
    "chain one own chunk", "chain two own chunks", "chain extra operand", "chain store_first=0",
}


def selector_instances() -> set:
    """Every (kernel, dtype, N, decode, tail N, CTAs) that select_conv_kernel_t / select_patch_kernel_t can return."""
    with open(os.path.join(CSRC, "conv_sm90.cu")) as f:
        conv = f.read()
    with open(os.path.join(CSRC, "conv3x3_patch_sm90.cu")) as f:
        patch = f.read()
    out = set()
    for dt in ("f16", "bf16"):
        for m in re.finditer(r"conv_wgmma_kernel<kBf16, (\d+), (true|false), (\d+), (\d+)>", conv):
            out.add(("conv", dt, int(m[1]), m[2] == "true", int(m[3]), int(m[4])))
        for m in re.finditer(r"conv3x3_patch_kernel<kBf16, (\d+), (\d+), (\d+)>", patch):
            out.add(("patch", dt, int(m[1]), False, int(m[2]), int(m[3])))
    return out


def _plans():
    for c in CASES:
        d, _ch = build_desc(c, fake_ptr)
        cfg = _C.conv_config(d)
        yield c, instance_key(c, d, cfg), plan_paths(c, cfg)


def test_case_names_are_unique():
    names = [c.name for c in CASES]
    assert len(names) == len(set(names))


def test_every_instance_is_reached():
    inst = selector_instances()
    assert len(inst) >= 54, sorted(inst)      # the patterns still match the selectors (27 instances per dtype today)
    reached = {}
    for c, key, _ in _plans():
        reached.setdefault(key, []).append(c.name)
    unknown = set(reached) - inst
    assert not unknown, f"cases planned onto instances the selectors do not list: {sorted(unknown)}"
    assert set(EXCLUDED) <= inst and not set(EXCLUDED) & set(reached)
    missing = inst - set(reached) - set(EXCLUDED)
    print(f"instance coverage: {len(inst & set(reached))} / {len(inst)} reached, {len(EXCLUDED)} excluded "
          f"({SMS} SMs)")
    for key in sorted(inst, key=str):
        print(f"  {key}: {reached[key][0] + (f' (+{len(reached[key]) - 1})' if len(reached[key]) > 1 else '') if key in reached else 'EXCLUDED: ' + EXCLUDED.get(key, 'MISSING')}")
    assert not missing, f"no case reaches {sorted(missing)}"


def test_every_plan_path_is_reached():
    seen = {}
    for c, _, paths in _plans():
        for p in paths:
            seen.setdefault(p, c.name)
    for p in sorted(REQUIRED_PATHS):
        print(f"  {p}: {seen.get(p, 'MISSING')}")
    assert REQUIRED_PATHS <= set(seen), sorted(REQUIRED_PATHS - set(seen))


def test_two_cta_threshold_at_2x_sms_tiles():
    """The same 1x1 layer plans two CTAs per SM at exactly 2 x SMs tiles and one CTA at one tile fewer."""
    by_name = {c.name: c for c in CASES}
    for dt in ("f16", "bf16"):
        for name, ctas, grid in ((f"{dt} 2cta 1x1 Cout32 at 2xSMs", 2, 2 * SMS), (f"{dt} 1cta 1x1 Cout32 at 2xSMs-1", 1, SMS)):
            c = by_name[name]
            d, _ = build_desc(c, fake_ptr)
            cfg = _C.conv_config(d)
            assert (cfg["ctas_per_sm"], cfg["grid"]) == (ctas, grid), (name, cfg)
