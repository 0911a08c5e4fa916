"""The case tables of tests/postprocess_cases.py reach every decode kernel instance, row-kernel branch, selection edge
and NMS branch of csrc/decode_nms.cu, and every branch of the fused decode epilogue (host logic, no GPU needed)."""
import conv_cases
from postprocess_cases import CASES, FUSED_CASES, fake_head_decode, fused_conv_case, fused_desc, fused_paths, \
    postprocess_paths
from yolort_b200 import _C

REQUIRED_PATHS = (
    # every decode kernel instance yb_decode_candidates launches
    {"rows f16", "rows bf16", "candidates f32", "candidates f16", "candidates bf16"}
    # the row kernel's branches
    | {"rows dense copy", "rows per-row copy", "rows warp straddles a level border", "rows partial last warp",
       "rows list overflow", "rows threshold 0", "rows 1 anchor", "rows 2 anchors", "rows 3 anchors", "rows 4 anchors",
       "rows W 1023"}
    # NHWC heads the row kernel must leave to the per-anchor kernel
    | {"nhwc W >= 1024 -> candidates", "nhwc H >= 1024 -> candidates", "nhwc row > 512 B -> candidates",
       "nhwc misaligned base -> candidates"}
    # the NMS kernel
    | {"sort bitonic R=4", "sort bitonic R=8", "sort radix", "nms trick", "nms trick, negative coordinates",
       "nms per-class labmask", "nms per-class no labmask", "nms explicit", "sweep multi-round", "sweep max_det stop",
       "max_det 1", "max_det 4096", "max_det 4096 reached", "rescale", "arena overflow in one image of a batch"}
    # the fused decode epilogue
    | {"fused f16", "fused bf16", "fused width 255", "fused width 256", "fused width 129", "fused width 192",
       "fused 4 anchors (a == 3)", "fused ragged M", "fused two levels in one arena"}
)

# Kernel instances no case reaches, with the test that compares them with the restatement.
EXCLUDED = {
    "decode_dense_kernel": "tests/test_gpu_logits_decoder.py::test_dense_decode_vs_oracle (fp32 / fp16 / bf16 against "
                           "oracle.restate.decode)",
    "decode_rows_kernel<TtaDecodeParams>": "tests/test_gpu_tta.py::test_multi_pass_decode_nms_vs_oracle (against "
                                           "oracle.restate_tta)",
}


def test_case_names_are_unique():
    names = [c.name for c in CASES] + [c.name for c in FUSED_CASES]
    assert len(names) == len(set(names))


def test_fused_cases_run_the_decode_instance():
    """Every fused case plans onto the conv kernel's fused-decode instance (conv_cases.EXCLUDED points here)."""
    for fc in FUSED_CASES:
        for level in range(len(fc.levels)):
            hd = fake_head_decode(fc)
            d = fused_desc(fc, level, conv_cases.fake_ptr, hd)
            key = conv_cases.instance_key(fused_conv_case(fc, level), d, _C.conv_config(d))
            assert key in conv_cases.EXCLUDED and "test_gpu_postprocess_paths" in conv_cases.EXCLUDED[key], (fc.name, key)


def test_every_path_is_reached():
    seen = {}
    for c in CASES:
        for p in postprocess_paths(c):
            seen.setdefault(p, []).append(c.name)
    for fc in FUSED_CASES:
        for p in fused_paths(fc):
            seen.setdefault(p, []).append(fc.name)
    print(f"post-processing path coverage: {len(REQUIRED_PATHS & set(seen))} / {len(REQUIRED_PATHS)} required paths, "
          f"{len(CASES)} + {len(FUSED_CASES)} cases")
    for p in sorted(REQUIRED_PATHS):
        print(f"  {p}: " + (f"{seen[p][0]}" + (f" (+{len(seen[p]) - 1})" if len(seen[p]) > 1 else "")
                            if p in seen else "MISSING"))
    for k, why in EXCLUDED.items():
        print(f"  excluded {k}: {why}")
    assert REQUIRED_PATHS <= set(seen), sorted(REQUIRED_PATHS - set(seen))
