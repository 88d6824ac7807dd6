"""The benchmarks under tools/: no tool imports another (shared code lives in tools/benchkit.py), every tool with a
command line starts without a GPU, benchkit's shared arithmetic gives the numbers each tool computed on its own before
it was shared (literals taken from those functions on the inputs below), and format_bench's table names real formats
and decoders and counts the algorithmic bytes the per-format scripts it replaced wrote."""
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


@pytest.mark.parametrize("name", ["yuv", "yuv_matrix", "yuv16", "yuv444", "bayer", "bayer16", "bayer_packed", "bf16"])
def test_format_bench_set_without_gpu(name, tmp_path):
    """Each set the per-format scripts ran is a --set of format_bench.py, which refuses to run it without a GPU and writes
    nothing."""
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, os.path.join(TOOLS, "format_bench.py"), "--out", str(tmp_path), "--set", name],
                       capture_output=True, text=True, env=env, timeout=300)
    assert r.returncode == 1 and "needs a CUDA device" in r.stderr, r.stderr
    assert not os.listdir(tmp_path)


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


def test_format_bench_arms():
    import format_bench as fb
    import kornia_rs_b200 as kb

    for name, s in fb.SETS.items():
        for section in (s.decode, s.pre, (("", s.e2e),)):
            for _, arms in section:
                for a in arms:
                    assert a.fmt in kb.SourceFormat.__members__, (name, a.label, a.fmt)
                    assert a.matrix is None or a.matrix in kb.YuvMatrix.__members__, (name, a.label, a.matrix)
        for _, arms in s.decode:
            for a in arms:
                assert callable(getattr(kb.imgproc, fb.decoder(fb.FMT[a.fmt]), None)), (name, a.label)


MATRICES = ("Bt601Limited", "Bt601Full", "Bt709Limited", "Bt709Full")
# the algorithmic bytes the eight per-format scripts this tool replaced wrote at 1080p, from results/h100_*_bench.jsonl
ALG_BYTES = {
    "yuv": {
        "yuv420_1080p_x256": {"Nv12": 2388787200, "Nv21": 2388787200, "I420": 2388787200, "Yv12": 2388787200},
        "yuv422_1080p_x256": {"Yuyv": 2654208000, "Uyvy": 2654208000, "Yvyu": 2654208000},
        "cfg3a_yuv420": {"Nv12": 7166361600, "I420": 7166361600, "Nv21": 7166361600, "Yv12": 7166361600},
        "cfg3b_yuv420": {"Nv12": 1759641600, "I420": 1759641600, "Nv21": 1759641600, "Yv12": 1759641600},
        "cfg3a_yuv422": {"Yuyv": 7431782400, "Uyvy": 7431782400},
        "cfg3b_yuv422": {"Yuyv": 1848115200, "Uyvy": 1848115200},
    },
    "yuv_matrix": {   # its line records no alg_bytes: n * (frame + 3 * w * h), n * (src + out bytes * dw * dh), 3b src = 1958400
        "nv12_1080p_x256": dict.fromkeys(MATRICES, 256 * (1920 * 1080 * 3 // 2 + 3 * 1920 * 1080)),
        "yuyv_1080p_x256": dict.fromkeys(MATRICES, 256 * (1920 * 1080 * 2 + 3 * 1920 * 1080)),
        "cfg3a_f32": dict.fromkeys(MATRICES, 256 * (1920 * 1080 * 3 // 2 + 12 * 1920 * 1080)),
        "cfg3a_f16": dict.fromkeys(MATRICES, 256 * (1920 * 1080 * 3 // 2 + 6 * 1920 * 1080)),
        "cfg3b_f32": dict.fromkeys(MATRICES, 256 * (1958400 + 12 * 640 * 640)),
        "cfg3b_f16": dict.fromkeys(MATRICES, 256 * (1958400 + 6 * 640 * 640)),
    },
    "yuv16": {
        "1080p_x256": {"P010": 4777574400, "P012": 4777574400, "I010": 4777574400, "I012": 4777574400, "Nv12": 2388787200, "Bayer12": 4246732800},
        "cfg3a_f32": {"P010": 7962624000, "P012": 7962624000, "I010": 7962624000, "I012": 7962624000, "Nv12": 7166361600, "Bayer12": 7431782400, "Bayer12_zeros": 7431782400},
        "cfg3a_f16": {"P010": 4777574400, "P012": 4777574400, "I010": 4777574400, "I012": 4777574400, "Nv12": 3981312000, "Bayer12": 4246732800, "Bayer12_zeros": 4246732800},
        "cfg3b_f32": {"P010": 2260992000, "P012": 2260992000, "I010": 2260992000, "I012": 2260992000, "Nv12": 1759641600, "Bayer12": 2319974400, "P010_generic": 2260992000},
        "cfg3b_f16": {"P010": 1631846400, "P012": 1631846400, "I010": 1631846400, "I012": 1631846400, "Nv12": 1130496000, "Bayer12": 1690828800, "P010_generic": 1631846400},
    },
    "yuv444": {
        "1080p_x256": {"I444": 3185049600, "I410": 6370099200, "I410Msb": 6370099200, "Nv12": 2388787200, "P010": 4777574400},
        "cfg3a_f32": {"I444": 7962624000, "I410": 9555148800, "I410Msb": 9555148800, "Nv12": 7166361600, "P010": 7962624000},
        "cfg3a_f16": {"I444": 4777574400, "I410": 6370099200, "I410Msb": 6370099200, "Nv12": 3981312000, "P010": 4777574400},
        "cfg3b_f32": {"I444": 1966080000, "I410": 2673868800, "I410Msb": 2673868800, "Nv12": 1759641600, "P010": 2260992000, "I444_generic": 1966080000},
        "cfg3b_f16": {"I444": 1336934400, "I410": 2044723200, "I410Msb": 2044723200, "Nv12": 1130496000, "P010": 1631846400, "I444_generic": 1336934400},
    },
    "bayer": {
        "1080p_x256": {"Nv12": 2388787200, "RGGB": 2123366400, "BGGR": 2123366400, "GRBG": 2123366400, "GBRG": 2123366400},
        "cfg3a": {"Nv12": 7166361600, "RGGB": 6900940800, "BGGR": 6900940800, "GRBG": 6900940800, "GBRG": 6900940800},
        "cfg3b": {"Nv12": 1759641600, "RGGB": 1789132800, "BGGR": 1789132800, "GRBG": 1789132800, "GBRG": 1789132800},
    },
    "bayer16": {
        "1080p_x256": {"Bayer12": 4246732800, "Bayer8": 2123366400, "Nv12": 2388787200},
        "cfg3a_f32": {"Bayer12": 7431782400, "Bayer8": 6900940800, "Nv12": 7166361600},
        "cfg3a_f16": {"Bayer12": 4246732800, "Bayer8": 3715891200, "Nv12": 3981312000},
        "cfg3b_f32": {"Bayer12": 2319974400, "Bayer8": 1789132800, "Nv12": 1759641600},
        "cfg3b_f16": {"Bayer12": 1690828800, "Bayer8": 1159987200, "Nv12": 1130496000},
    },
    "bayer_packed": {
        "1080p_x256": {"Raw10p": 3848601600, "Raw12p": 3981312000, "Raw14p": 4114022400, "Bayer12": 4246732800, "Raw12p_generic": 3981312000},
        "cfg3a_f32": {"Raw10p": 7033651200, "Raw12p": 7166361600, "Raw14p": 7299072000, "Bayer12": 7431782400, "Raw12p_generic": 7166361600},
        "cfg3a_f16": {"Raw10p": 3848601600, "Raw12p": 3981312000, "Raw14p": 4114022400, "Bayer12": 4246732800, "Raw12p_generic": 3981312000},
        "cfg3b_f32": {"Raw10p": 1921843200, "Raw12p": 2054553600, "Raw14p": 2187264000, "Bayer12": 2319974400},
        "cfg3b_f16": {"Raw10p": 1292697600, "Raw12p": 1425408000, "Raw14p": 1558118400, "Bayer12": 1690828800},
    },
    "bf16": {
        "Nv12_cfg3a": {"f32": 7166361600, "f16": 3981312000, "bf16": 3981312000},
        "Nv12_cfg3b": {"f32": 1759641600, "f16": 1130496000, "bf16": 1130496000},
        "P010_cfg3a": {"f32": 7962624000, "f16": 4777574400, "bf16": 4777574400},
        "P010_cfg3b": {"f32": 2260992000, "f16": 1631846400, "bf16": 1631846400},
        "BayerRggb12_cfg3a": {"f32": 7431782400, "f16": 4246732800, "bf16": 4246732800},
        "BayerRggb12_cfg3b": {"f32": 1730150400, "f16": 1101004800, "bf16": 1101004800},
        "I444_cfg3a": {"f32": 7962624000, "f16": 4777574400, "bf16": 4777574400},
        "I444_cfg3b": {"f32": 1966080000, "f16": 1336934400, "bf16": 1336934400},
        "Yuyv_cfg3a": {"f32": 7431782400, "f16": 4246732800, "bf16": 4246732800},
        "Yuyv_cfg3b": {"f32": 1730150400, "f16": 1101004800, "bf16": 1101004800},
        "Nv12_cfg3b_lanczos": {"f32": 2054553600, "f16": 1425408000, "bf16": 1425408000},
    },
}


@pytest.mark.parametrize("name", sorted(ALG_BYTES))
def test_format_bench_alg_bytes(name):
    import format_bench as fb

    s = fb.SETS[name]
    got = {key: {a.label: fb.decode_bytes(a, w, h, n) for a in arms} for key, w, h, n, arms in fb.decode_sections(s) if w == 1920}
    for group, arms in s.pre:
        got.update({key: {a.label: fb.pre_bytes(a, cfg, out) for a in arms_c} for key, cfg, out, arms_c in fb.pre_sections(s, group, arms)})
    assert got == ALG_BYTES[name]
