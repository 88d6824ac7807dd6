"""Camera preprocess: a seeded sweep of random geometries and descriptors over every source format, kernel, sampler and
entry, against references that do not use the library's decoders.

`case(i)` is a pure function of its index (numpy.random.default_rng(BASE + i)): format i % 51, descriptor kind
(i // 51) % 9, and random source size, pitch padding, destination size, sampler, output type, entry, frame layout,
YUV matrix and normalisation.  Hand-picked edge cases (EDGES) run through the same machinery.  Each case:

  * runs through its entry (pointer table, strided, or host pipeline) into a destination prefilled with 0xFF bytes (NaN in
    f32 and f16) inside harness.Guarded, whose guards must keep their fill;
  * must run the kernel that `expected_kernel`, a host mirror of launch_preprocess's dispatch rule, names for it;
  * is compared with a restatement the suite already trusts: the oracle's ko_preprocess_frame on the case's own
    descriptor (for YUV and Bayer frames on the restated RGB8 decode), or restate.preprocess_rgb16 on the restated
    16-bit RGB decode; bit for bit, Lanczos within the oracle tolerance (host sinf against CUDA's);
  * unless it samples with Lanczos, runs a second time into a destination one element past a 16-byte boundary, which
    refuses the identity and fast kernels: the generic kernel must then give the same bits.

test_sweep_coverage (CPU only) runs every case through the dispatch mirror and asserts what the sweep covers, so that a
change to the generator cannot silently shrink it.
"""
import ctypes as C
from collections import defaultdict
from dataclasses import dataclass

import numpy as np
import pytest
import torch

from harness import Guarded, dev, lib
from restate import BILINEAR, EDGES, ENTRIES, FORMATS, GENERIC, IMAGENET_INV, KINDS, LANCZOS, MATRICES, NEAREST, NORMS, N_SWEEP, SAMPLING_NAME, case, decode_yuv16, decode_yuv444, decode_yuv444_16, decode_yuv8, demosaic, expected_kernel, frame_bytes, group, host_chunk, oracle_rgb, preprocess_rgb16, row_bytes, to_twin, unpack, yuv


def reference(c, raw):
    """(3, dh, dw) expected output of one frame: f16 bits, or f32 (Lanczos: always f32, compared within a tolerance)."""
    f, w, h = c.fmt, c.w, c.h
    h16 = c.f16 and c.sampling != LANCZOS
    m = MATRICES[c.matrix]
    rows = raw[:c.pitch * h].reshape(h, c.pitch)[:, :row_bytes(f, w, c.bpp)]
    if f.family in ("rgb", "gray"):
        return oracle_rgb(c, raw, c.code, c.bpp, c.pitch, h16)
    if f.family in ("yuv420", "yuv422") and not f.words:
        tight = raw if f.family == "yuv420" else np.ascontiguousarray(rows).reshape(-1)
        if c.matrix == 0:   # BT.601 limited: the oracle reads NV12 and YUYV itself
            twin = to_twin(tight, w, h, f.layout)
            return oracle_rgb(c, twin, 3 if f.family == "yuv420" else 4, 1 if f.family == "yuv420" else 2, w if f.family == "yuv420" else 2 * w, h16)
        rgb = decode_yuv8(tight, w, h, f.layout, m)
    elif f.code == 11:
        rgb = decode_yuv444(raw, w, h, m)
    elif f.family == "bayer" and not f.words and not f.packed:
        rgb = demosaic(np.ascontiguousarray(rows), f.layout).astype(np.uint8)
    else:
        if f.family == "bayer":
            samples = np.ascontiguousarray(rows).view("<u2") if f.words else unpack(np.ascontiguousarray(rows), f.bits)
            rgb16 = demosaic(np.asarray(samples).astype(np.uint16), f.layout)
        else:
            words = torch.from_numpy(raw.view("<u2").astype(np.int32))
            rgb16 = (decode_yuv16 if f.family == "yuv420" else decode_yuv444_16)(words, w, h, f.name, m).numpy()
        mean, inv = NORMS[c.norm]
        return preprocess_rgb16(np.asarray(rgb16).astype(np.uint16), f.bits, (c.scale_x, c.scale_y, c.pad_x, c.pad_y), c.dw, c.dh,
                                SAMPLING_NAME[c.sampling], mean, inv, c.pad_value, h16)
    return oracle_rgb(c, np.ascontiguousarray(rgb), 0, 3, 3 * w, h16)


def compare(got, want, c, what):
    if c.sampling == LANCZOS:
        # host sinf against CUDA's: the oracle's f32 tolerance, scaled with the normalisation's gain, plus for f16 output one
        # f16 step at the expected value (the kernel rounds its own f32 result, which may sit across a binade boundary from the
        # oracle's; Lanczos overshoot passes 256 at gain 255).  At ImageNet gain that is the oracle's 2e-3.
        g = got.view(np.float16 if c.f16 else np.float32).astype(np.float32)
        want = want.reshape(-1).astype(np.float32)
        tol = 1e-4 * max(1.0, max(NORMS[c.norm][1]) / max(IMAGENET_INV)) + (np.spacing(np.abs(want).astype(np.float16)).astype(np.float32)
                                                                             if c.f16 else 0.0)
        over = np.abs(g - want) - tol
        assert over.max() <= 0, f"{what}: error {float(np.abs(g - want)[over.argmax()])} at element {int(over.argmax())} exceeds {float(np.broadcast_to(tol, over.shape)[over.argmax()])}"
    else:
        w = np.ascontiguousarray(want).reshape(-1).view(np.uint8)
        bad = np.flatnonzero(got != w)
        assert bad.size == 0, f"{what}: {bad.size} bytes differ, first at byte {bad[0]}"


# ── the GPU run ─────────────────────────────────────────────────────────────────────────────────────────────────────
def run_case(kb, lib, dev, c):
    from kornia_rs_b200._lib import PreprocessDesc
    f = c.fmt
    d = c.desc(PreprocessDesc)
    need = c.need
    assert lib.kb200_preprocess_src_bytes(C.byref(d)) == need, str(c)
    if c.kind in ("letterbox", "stretch"):
        a = (C.c_float * 4)()
        lib.kb200_preprocess_affine(KINDS.index(c.kind), c.w, c.h, c.dw, c.dh, a)
        assert tuple(a) == (c.scale_x, c.scale_y, c.pad_x, c.pad_y), str(c)
    frames = [frame_bytes(c, k) for k in range(c.batch)]
    esz = 2 if c.f16 else 4
    out_elems = 3 * c.dw * c.dh
    nbytes = out_elems * esz * c.batch
    starts = list(c.frames) if c.entry == "table" else [c.frames[0] + k * c.stride for k in range(c.batch)]
    span = starts[-1] + need
    image = np.zeros(span, np.uint8)
    for s, fr in zip(starts, frames):
        image[s:s + need] = fr
    dev_src = Guarded(dev, span).load("u8", image)
    host_src = Guarded(dev, span, host=True).load("u8", image) if c.entry == "host" else None
    fn = {(e, h): getattr(lib, f"kb200_preprocess{'_strided' if e == 'strided' else ''}_{'f16' if h else 'f32'}") for e in ("table", "strided") for h in (0, 1)}

    def device_call(entry, dst):
        if entry == "table":
            ptrs = (C.c_void_p * c.batch)(*[dev_src.ptr + s for s in starts])
            lens = (C.c_size_t * c.batch)(*[need] * c.batch)
            st = fn["table", c.f16](None, C.byref(d), ptrs, lens, c.batch, dst.ptr, out_elems * c.batch)
            return st, expected_kernel(d, [dev_src.ptr + s for s in starts], None, dst.ptr, c.sampling)
        st = fn["strided", c.f16](None, C.byref(d), dev_src.ptr + c.frames[0], dev_src.n - c.frames[0], c.stride, c.batch, dst.ptr, out_elems * c.batch)
        return st, expected_kernel(d, [dev_src.ptr + c.frames[0]], c.stride, dst.ptr, c.sampling)

    outs = []
    runs = [(0, c.planned())] + ([(esz, GENERIC)] if c.sampling != LANCZOS else [])
    for off, want_kernel in runs:
        host = c.entry == "host" and off == 0
        dst = Guarded(dev, nbytes, min(nbytes, 1 << 16), off, host=host).fill(0xFF)
        if host:
            _, src_chunk, dst_chunk = host_chunk(need, out_elems * esz, c.batch)
            pipe = kb.imgproc.HostPipeline(dev, src_chunk_bytes=src_chunk, dst_chunk_bytes=dst_chunk, depth=2)
            try:
                st = lib.kb200_preprocess_host(pipe._h, None, C.byref(d), host_src.ptr + c.frames[0], host_src.n - c.frames[0], c.stride, c.batch,
                                               dst.ptr, out_elems * c.batch, int(c.f16))
                mirror = c.planned()
                torch.cuda.synchronize()
            finally:
                pipe.close()
        else:
            st, mirror = device_call("table" if c.entry == "table" else "strided", dst)
        assert st == 0, f"{c}: status {st}: {kb._lib.last_error()}"
        ran = kb._lib.last_kernel()
        torch.cuda.synchronize()
        assert ran == want_kernel == mirror, f"{c}: dst +{off} B ran {ran}, the dispatch mirror says {mirror}, the case plans {want_kernel}"
        lead, tail = dst.guards()
        for what, g in (("lead", lead), ("tail", tail)):
            bad = np.flatnonzero(g != 0xFF)
            assert bad.size == 0, f"{c}: dst +{off} B: {bad.size} bytes written in the {what} guard"
        outs.append(dst.out())
    ones = outs[0].view(np.uint16 if c.f16 else np.uint32) == (0xFFFF if c.f16 else 0xFFFFFFFF)
    assert not ones.any(), f"{c}: {int(ones.sum())} output elements left unwritten (first {int(np.flatnonzero(ones)[0])})"
    fb = out_elems * esz
    check = range(c.batch) if c.batch <= 4 else sorted({0, 1, 255, 256, c.batch - 1})
    for k in check:
        compare(outs[0][k * fb:(k + 1) * fb], reference(c, frames[k]), c, f"{c}: frame {k} differs from the reference")
    if len(outs) == 2:
        bad = np.flatnonzero(outs[0] != outs[1])
        assert bad.size == 0, f"{c}: {c.planned()} and {GENERIC} differ in {bad.size} bytes, first at byte {bad[0]} (frame {bad[0] // fb})"


@pytest.mark.gpu
@pytest.mark.parametrize("i", range(N_SWEEP))
def test_sweep(kb, lib, dev, i):
    run_case(kb, lib, dev, case(i))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(EDGES))
def test_edge(kb, lib, dev, name):
    run_case(kb, lib, dev, EDGES[name])


# ── what the sweep covers (CPU) ─────────────────────────────────────────────────────────────────────────────────────
def straddles(bits, w):
    """A packed identity thread at column x reads bits / 2 bytes from x * bits / 8: past its 8-byte word at some x."""
    return any(((x * bits // 8) & 7) + bits // 2 > 8 for x in range(0, w, 4))


def test_sweep_coverage():
    cases = [case(i) for i in range(N_SWEEP)] + list(EDGES.values())
    assert len({c.name for c in cases}) == len(cases)
    kernels, samplers, matrices, kinds = defaultdict(set), defaultdict(set), defaultdict(set), set()
    entries, outs, dst_w4, fast_h8, split = set(), set(), set(), set(), set()
    bayer_id = defaultdict(set)
    for c in cases:
        f = c.fmt
        k = c.planned()
        assert c.planned(dst=16 + (2 if c.f16 else 4)) == GENERIC or c.entry == "host"
        kernels[c.code].add(k)
        samplers[group(f)].add(c.sampling)
        if yuv(f):
            matrices[group(f)].add(c.matrix)
        kinds.add(c.kind.split("-")[0])
        entries.add(c.entry)
        outs.add(c.f16)
        dst_w4.add(c.dw % 4)
        if k == f.fast:
            fast_h8.add(c.dh % 8)
        if c.batch > 256:
            split.add("identity" if k == f.identity else "fast" if k == f.fast else "generic")
        if f.family == "bayer" and k == f.identity:
            t = group(f)
            bayer_id[t] |= {f"h{c.h % 2}", *(["h=3"] if c.h == 3 else []), *(["w=4"] if c.w == 4 else [])}
            if f.packed and straddles(f.bits, c.w):
                bayer_id[t].add("straddle")
    for code, f in FORMATS.items():
        assert kernels[code] == {k for k in (f.identity, f.fast, GENERIC) if k}, f"{f.name}: ran {sorted(kernels[code])}"
    for g in {group(f) for f in FORMATS.values()}:
        assert samplers[g] == {NEAREST, BILINEAR, LANCZOS}, g
    for g in {group(f) for f in FORMATS.values() if yuv(f)}:
        assert matrices[g] == {0, 1, 2, 3}, g
    assert kinds == {k.split("-")[0] for k in KINDS}, kinds
    assert entries == set(ENTRIES) and outs == {False, True}
    assert dst_w4 == {0, 1, 2, 3}
    assert fast_h8 == set(range(8)), fast_h8
    assert split == {"identity", "fast", "generic"}, split
    for t in ("bayer8", "bayer16", "bayer10p", "bayer12p", "bayer14p"):
        want = {"h0", "h1", "h=3", "w=4"} | ({"straddle"} if t.endswith("p") else set())
        assert bayer_id[t] >= want, (t, bayer_id[t])
