#!/usr/bin/env python
"""Extracts the reference's OWN CUDA kernel strings into baseline/_ref/ — the GPU baseline of SURVEY §8(d) / BASELINE.md §2.

The reference (kornia-rs) ships its GPU kernels as CUDA-C source strings inside Rust files and JIT-compiles them with
NVRTC for `compute_XY` with `--fmad=false` (crates/kornia-tensor/src/cuda.rs:675-718).  This script reads those strings
from a kornia-rs checkout (the directory $KORNIA_RS_SRC names) *where they lie*, compiles each NVRTC translation unit
IN MEMORY exactly like the reference does on an H100
(NVRTC, `--gpu-architecture=compute_90 --fmad=false`, nothing else) to `baseline/_ref/ptx/<unit>.ptx`, and records a
manifest (unit -> reference file:line, kernel names).  Only the compiled PTX is kept — the source text is never written
into the repository tree; `baseline/_ref/` is git-ignored like a built .so.
`baseline/ref_gpu.py` loads the PTX through the driver API and launches it with the reference's launch geometry.  Test / measurement infrastructure only: nothing here is
linked into, imported by or shipped with the product library.

Run by `__graft_entry__.build()` whenever $KORNIA_RS_SRC is set.
"""
from __future__ import annotations

import json
import os
import re
import sys

REF = os.path.join(os.environ.get("KORNIA_RS_SRC", ""), "crates", "kornia-imgproc", "src")
HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_ref")


def raw_strings(text: str) -> list[tuple[int, str]]:
    """All Rust raw string literals r#"..."# of `text` as (line, body)."""
    return [(text.count("\n", 0, m.start()) + 1, m.group(1)) for m in re.finditer(r'r#"(.*?)"#', text, re.S)]


def static_str(text: str, name: str) -> tuple[int, str]:
    m = re.search(r"(?:static|const)\s+" + re.escape(name) + r'\s*:\s*&str\s*=\s*r#"(.*?)"#\s*;', text, re.S)
    if not m:
        raise KeyError(name)
    return text.count("\n", 0, m.start()) + 1, m.group(1)


def fn_body(text: str, fn: str) -> tuple[int, str]:
    """Source text of a top-level Rust `fn` (from its signature to the first line that is a lone `}`)."""
    m = re.search(r"^(?:pub(?:\([a-z]+\))?\s+)?fn\s+" + re.escape(fn) + r"\b", text, re.M)
    if not m:
        raise KeyError(fn)
    end = re.compile(r"^\}\s*$", re.M).search(text, m.end())
    return text.count("\n", 0, m.start()) + 1, text[m.start():end.end()]


def rust_format(template: str, **fields) -> str:
    """Rust `format!` semantics for named arguments: {name} substituted, {{ and }} are literal braces."""
    out, i = [], 0
    while i < len(template):
        c = template[i]
        if template.startswith("{{", i):
            out.append("{"); i += 2
        elif template.startswith("}}", i):
            out.append("}"); i += 2
        elif c == "{":
            j = template.index("}", i)
            out.append(str(fields[template[i + 1:j]]))
            i = j + 1
        else:
            out.append(c); i += 1
    return "".join(out)


def sep_f32_unit(text: str, channels: int, ktaps: int, horizontal: bool) -> tuple[int, str, str]:
    """cuda/filter.rs `sep_f32_src(channels, ktaps, horizontal)` evaluated here (the Rust fn is a format! template)."""
    line, body = fn_body(text, "sep_f32_src")
    strs = [s for _, s in raw_strings(body)]
    coord_h, coord_v, template = strs[0], strs[1], strs[2]
    loop_head, bound = ("#pragma unroll", f"{ktaps}u") if ktaps > 0 else ("", "ktaps")   # unroll_prelude()
    axis = "h" if horizontal else "v"
    src = rust_format(template, channels=channels, ktaps=ktaps, axis=axis, loop_head=loop_head, bound=bound,
                      coord=coord_h if horizontal else coord_v)
    return line, f"sep_filter_f32_{axis}_c{channels}_k{ktaps}", src


def units() -> list[dict]:
    """One entry per NVRTC translation unit the reference compiles on the §8 path."""
    out = []

    def add(unit, rs, line, src, kernels):
        out.append({"unit": unit, "rs": rs, "line": line, "src": src, "kernels": kernels})

    def statics(rs, specs, prelude=None):
        text = open(os.path.join(REF, rs)).read()
        for unit, names, kernels in specs:
            parts, first = [], None
            if prelude:   # get_kernel(): format!("{CUDA_COLOR_COMMON}\n{src}")   (cuda/color/mod.rs:186-200)
                parts.append(static_str(open(os.path.join(REF, prelude[0])).read(), prelude[1])[1])
            for n in names:
                line, s = static_str(text, n)
                first = first or line
                parts.append(s)
            add(unit, rs, first, "\n".join(parts), kernels)

    statics("cuda/resize.rs", [
        ("resize_bilinear", ["BILINEAR_SRC"], ["resize_bilinear_downscale_3c"]),
        ("resize_nearest", ["NEAREST_SRC"], ["resize_nearest_downscale_3c"]),
        ("resize_bilinear_normalize", ["BILINEAR_NORMALIZE_SRC"], ["resize_bilinear_normalize_3c"]),
        ("resize_bicubic", ["BICUBIC_SRC"], ["resize_bicubic_3c"]),
        ("resize_lanczos_h", ["LANCZOS_H_SRC"], ["resize_lanczos_h_3c"]),
        ("resize_lanczos_v", ["LANCZOS_V_SRC"], ["resize_lanczos_v_3c"]),
    ])
    statics("cuda/warp_perspective.rs", [
        ("warp_perspective_bilinear", ["BILINEAR_SRC"], ["warp_perspective_bilinear_3c"]),
        ("warp_perspective_nearest", ["NEAREST_SRC"], ["warp_perspective_nearest_3c"]),
        ("warp_perspective_bicubic", ["BICUBIC_SRC"], ["warp_perspective_bicubic_3c"]),
        ("warp_perspective_lanczos", ["LANCZOS_SRC"], ["warp_perspective_lanczos_3c"]),
    ])
    statics("cuda/warp_affine.rs", [
        ("warp_affine_bilinear", ["BILINEAR_SRC"], ["warp_affine_bilinear_3c"]),
        ("warp_affine_nearest", ["NEAREST_SRC"], ["warp_affine_nearest_3c"]),
        ("warp_affine_bicubic", ["BICUBIC_SRC"], ["warp_affine_bicubic_3c"]),
        ("warp_affine_lanczos", ["LANCZOS_SRC"], ["warp_affine_lanczos_3c"]),
    ])
    statics("cuda/remap.rs", [
        ("remap_bilinear", ["BILINEAR_SRC"], ["remap_bilinear_3c"]),
        ("remap_nearest", ["NEAREST_SRC"], ["remap_nearest_3c"]),
    ])
    statics("cuda/color/gray.rs", [
        ("gray_from_rgb_f32", ["GRAY_FROM_RGB_F32_SRC"], ["gray_from_rgb_f32"]),
        ("gray_from_rgb_u8", ["GRAY_FROM_RGB_U8_SRC"], ["gray_from_rgb_u8"]),
    ], prelude=("cuda/color/mod.rs", "CUDA_COLOR_COMMON"))
    statics("cuda/color/video.rs", [
        # PLANAR420_SRC / PACKED422_SRC = format!("{DECODE_COMMON}\n{..._TAIL}")   (cuda/color/video.rs:280-283)
        ("rgb_from_planar420", ["DECODE_COMMON", "PLANAR420_SRC_TAIL"], ["rgb_from_planar420_u8"]),
        ("rgb_from_packed422", ["DECODE_COMMON", "PACKED422_SRC_TAIL"], ["rgb_from_packed422_u8"]),
    ], prelude=("cuda/color/mod.rs", "CUDA_COLOR_COMMON"))
    statics("cuda/filter.rs", [("gradient_magnitude", ["MAGNITUDE_SRC"], ["gradient_magnitude_f32"])])
    statics("preprocess.rs", [
        ("preprocess", ["KERNEL_SRC"], ["resize_normalize_to_chw_bilinear", "resize_normalize_to_chw_nearest",
                                        "resize_normalize_to_chw_lanczos", "resize_normalize_to_chw_bilinear_f16",
                                        "resize_normalize_to_chw_nearest_f16", "resize_normalize_to_chw_lanczos_f16"]),
    ])
    ftext = open(os.path.join(REF, "cuda/filter.rs")).read()
    for c in (1, 3, 4):
        for k in (3, 5, 7):
            for horizontal in (True, False):
                line, name, src = sep_f32_unit(ftext, c, k, horizontal)
                add(name, "cuda/filter.rs", line, src, [name])
    return out


def nvrtc_ptx(src: str, name: str) -> bytes:
    """NVRTC with the reference's two options (kornia-tensor/src/cuda.rs:703-718): arch + fmad=false."""
    from cuda.bindings import nvrtc

    def ck(r):
        if r[0] != nvrtc.nvrtcResult.NVRTC_SUCCESS:
            raise RuntimeError(f"nvrtc: {r[0]}")
        return r[1:] if len(r) > 2 else (r[1] if len(r) == 2 else None)

    prog = ck(nvrtc.nvrtcCreateProgram(src.encode(), f"{name}.cu".encode(), 0, [], []))
    opts = [b"--gpu-architecture=compute_90", b"--fmad=false"]
    res = nvrtc.nvrtcCompileProgram(prog, len(opts), opts)
    if res[0] != nvrtc.nvrtcResult.NVRTC_SUCCESS:
        n = ck(nvrtc.nvrtcGetProgramLogSize(prog))
        log = b" " * n
        nvrtc.nvrtcGetProgramLog(prog, log)
        raise RuntimeError(f"NVRTC failed for {name}:\n{log.decode(errors='replace')}")
    n = ck(nvrtc.nvrtcGetPTXSize(prog))
    ptx = b" " * n
    ck(nvrtc.nvrtcGetPTX(prog, ptx))
    nvrtc.nvrtcDestroyProgram(prog)
    return ptx


def main() -> int:
    if not os.path.isdir(REF):
        print(f"[ref-kernels] {REF} not present: keeping whatever baseline/_ref already holds")
        return 0
    import shutil

    shutil.rmtree(os.path.join(OUT, "kernels"), ignore_errors=True)     # source text is never kept: only the compiled PTX
    os.makedirs(os.path.join(OUT, "ptx"), exist_ok=True)
    manifest = {}
    for u in units():
        ptx = nvrtc_ptx(u["src"], u["unit"])
        with open(os.path.join(OUT, "ptx", u["unit"] + ".ptx"), "wb") as f:
            f.write(ptx)
        manifest[u["unit"]] = {"source": f"crates/kornia-imgproc/src/{u['rs']}:{u['line']}", "kernels": u["kernels"]}
    with open(os.path.join(OUT, "manifest.json"), "w") as f:
        json.dump({"nvrtc_options": ["--gpu-architecture=compute_90", "--fmad=false"], "units": manifest}, f, indent=1)
    print(f"[ref-kernels] {len(manifest)} NVRTC units extracted from {REF} and compiled to PTX under {OUT}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
