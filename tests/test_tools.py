"""The benchmarks under tools/: no tool imports another (shared code lives in tools/benchkit.py), every tool with a
command line starts without a GPU, and benchkit's shared arithmetic gives the numbers each tool computed on its own
before it was shared (literals taken from those functions on the inputs below)."""
import ast
import glob
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOOLS = os.path.join(ROOT, "tools")
sys.path.insert(0, TOOLS)

import benchkit  # noqa: E402

F32 = np.float32
W, H = 64, 48
SCRIPTS = sorted(glob.glob(os.path.join(TOOLS, "*.py")))
TOOL_NAMES = {os.path.basename(p)[:-3] for p in SCRIPTS}


def imported_modules(path):
    mods = set()
    for n in ast.walk(ast.parse(open(path).read())):
        if isinstance(n, ast.Import):
            mods |= {a.name.split(".")[0] for a in n.names}
        elif isinstance(n, ast.ImportFrom) and n.level == 0:
            mods.add(n.module.split(".")[0])
    return mods


def test_no_tool_imports_another():
    for path in SCRIPTS:
        name = os.path.basename(path)[:-3]
        allowed = set() if name == "benchkit" else {"benchkit"}
        assert not (imported_modules(path) & TOOL_NAMES) - allowed, f"{name} imports {(imported_modules(path) & TOOL_NAMES) - allowed}"


def has_command_line(path):
    return any(isinstance(n, ast.Call) and getattr(n.func, "id", getattr(n.func, "attr", None)) == "parse_args"
               for n in ast.walk(ast.parse(open(path).read())))


@pytest.mark.parametrize("script", [os.path.basename(p) for p in SCRIPTS if has_command_line(p) and not p.endswith("benchkit.py")])
def test_tool_help_without_gpu(script):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, os.path.join(TOOLS, script), "--help"], capture_output=True, text=True, env=env, timeout=300)
    assert r.returncode == 0, r.stderr
    assert "--out" in r.stdout


def np_inverse(fwd):
    m = np.array(fwd, np.float64).reshape(3, 3)
    persp = not (m[2, 0] == 0.0 and m[2, 1] == 0.0 and m[2, 2] == 1.0)
    inv = np.linalg.inv(m).astype(F32)
    if not persp:
        inv[2] = (0.0, 0.0, 1.0)
    return inv, persp


def warp_regions():
    from restate import forward_of

    ang = np.random.default_rng(7).uniform(-0.6, 0.6)
    rot = np.array([[np.cos(ang), -np.sin(ang), 20.0], [np.sin(ang), np.cos(ang), 10.0], [0, 0, 1]])
    persp = np.array([[1.1, 0.2, 5.0], [0.05, 0.9, 7.0], [1e-3, -2e-3, 1.0]])
    corner = np.array([[1.3, 0.0, 44.0], [0.0, 1.3, 33.0], [0, 0, 1]])   # reaches x = 63.5, y = 47.3: the last column and row
    whole = np.array([[4.0, 0.0, 0.0], [0.0, 4.0, 0.0], [0, 0, 1]])      # integer taps only, past the frame's edge
    return [(0, forward_of(rot)), (0, forward_of(corner)), (1, forward_of(persp)), (1, forward_of(whole))]


def remap_map():
    rng = np.random.default_rng(11)
    mx = rng.uniform(-4, W + 4, (12, 16)).astype(F32)
    my = rng.uniform(-4, H + 4, (12, 16)).astype(F32)
    mx[0, :4] = (np.nan, np.inf, -np.inf, 3.5)
    my[0, :4] = (2.0, 5.0, 7.0, np.nan)
    mx[1, :3] = (W - 0.5, W - 1, 10.25)   # the last column, with and without a second tap
    my[1, :3] = (H - 0.25, 20.0, H - 1)   # the last row
    mx[2, 0], my[2, 0] = np.inf, -np.inf
    return mx, my


def test_warp_tapped_bytes():
    import preprocess_warp_bench as pw

    want = {"NV12": 1704, "P010": 3408, "RGGB": 2406}
    assert {f: pw.tapped_bytes(f, W, H, warp_regions(), np_inverse, 16, 12) for f in want} == want
    assert {f: benchkit.frame_len(f, W, H) for f in want} == {"NV12": 4608, "P010": 9216, "RGGB": 3072}


def test_remap_tapped_bytes():
    import preprocess_remap_bench as pr

    mx, my = remap_map()
    want = {"NV12": 968, "P010": 1936, "RGGB12": 2962}
    assert {f: pr.tapped_bytes(f, W, H, mx, my) for f in want} == want
    assert benchkit.frame_len("RGGB12", W, H) == 6144


ROW_ARGS = ({"Nv12": [1.2345678, 1.1000049, 1.3], "RGGB": [2.0, 2.5, 2.25]}, {"Nv12": "nv12_kernel", "RGGB": "bayer_kernel"},
            {"Nv12": 123456789, "RGGB": 98765432}, {"Nv12": None, "RGGB": True})


@pytest.mark.parametrize("check_key", ["bit_identical_to_sibling", "output_checked"])
def test_row(check_key):
    assert benchkit.row(*ROW_ARGS, check_key) == {
        "Nv12": {"ms": [1.2346, 1.1, 1.3], "ms_min": 1.1, "alg_bytes": 123456789, "gbs": 112.2, "frac_of_3350": 0.034, "kernel": "nv12_kernel",
                 check_key: None},
        "RGGB": {"ms": [2.0, 2.5, 2.25], "ms_min": 2.0, "alg_bytes": 98765432, "gbs": 49.4, "frac_of_3350": 0.015, "kernel": "bayer_kernel",
                 check_key: True}}


def test_e2e_result():
    steps, transfer = [31.41592, 27.18281, 29.0], (123456789, 987654321)
    want = {"ms_per_step": [31.416, 27.183, 29.0], "ms_min": 27.183, "h2d_bytes": 123456789, "d2h_bytes": 987654321, "h2d_gbs": 4.5,
            "d2h_gbs": 36.3}
    assert benchkit.e2e_result(steps, transfer, False) == {**want, "matches_device_result": False}
    assert benchkit.e2e_result(steps, transfer, True, pixels=64 * 1280 * 720) == {**want, "gpix_s": 2.17, "matches_device_result": True}
    assert benchkit.e2e_result(steps, transfer) == want


def test_share_of_peak_rounding():
    rng = np.random.default_rng(3)
    for nbytes, ms in zip(rng.integers(1, 10**11, 2000), rng.uniform(0.01, 100.0, 2000)):
        nbytes = int(nbytes)
        assert round(nbytes / (ms * 1e-3) / (benchkit.PEAK_GBS * 1e9), 3) == round(nbytes / (ms * 1e-3) / 3.35e12, 3)
