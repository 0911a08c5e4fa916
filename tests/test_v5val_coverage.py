"""The case tables of tests/v5val_cases.py reach every INTER_AREA path, load_image branch, letterbox mode and pad
parity, rect-block branch, the P6 stride and a partial last batch (host logic, no GPU needed)."""
import v5val_cases as C

REQUIRED_PATHS = (
    {"area general", "area 2x2", "area other integer", "linear up-scale", "no resize"}
    | {"letterbox resize, auto", "letterbox resize, scale_fill"}
    | {f"{k} pad {side}" for k in ("odd", "zero") for side in ("top", "bottom", "left", "right")}
    | {f"letterbox {k} pad {side}" for k in ("odd", "zero") for side in ("top", "bottom", "left", "right")}
    | {"portrait batch", "landscape batch", "mixed batch"}
    | {"stride 64", "partial last batch"}
)


def test_case_tables_reach_every_path():
    missing = REQUIRED_PATHS - C.paths()
    assert not missing, sorted(missing)
