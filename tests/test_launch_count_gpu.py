"""The kernel_launches counter of a context (cfb_context_stats) against a torch.profiler trace of the same call: every
entry point counts exactly the kernels it launched.  Covers every encode source at level masks 1 and 7, at a width of
whole lanes and at one whose level-2 / level-3 planes are ragged (edge kernels); both interlaced modes; every decode
output at every resolution it supports; the two-frame GOP; the free-standing level; the temporal and sparse entry points."""
import importlib
import json
import os
import tempfile

import numpy as np
import pytest

from gpu_fixtures import ctx  # noqa: F401

pytestmark = pytest.mark.gpu

PKG = importlib.import_module("cineform-sdk_b200")
P, I, HL = PKG.PROGRESSIVE, PKG.INTERLACED, PKG.INTERLACED_HL_INTEGRATED
FULL, HALF, QUARTER = PKG.RESOLUTION_FULL, PKG.RESOLUTION_HALF, PKG.RESOLUTION_QUARTER
H = 96

# source -> (width of whole lanes at every level, width with ragged level-2 / level-3 planes)
_WIDTHS = {"YUYV": (384, 400), "UYVY": (384, 400), "YU64": (384, 400), "V210": (384, 432),
           "PLANAR16": (384, 392), "RG48": (384, 392), "RG30": (384, 392), "AB10": (384, 392), "AR10": (384, 392),
           "R210": (384, 392), "DPX0": (384, 392), "B64A": (384, 392), "RG64": (384, 392),
           "BYR4": (384, 208), "BYR5": (384, 208)}
_422 = ("YUYV", "UYVY", "YU64", "V210")

# (codec source, frame flags, output, {resolution: interlaced modes})
_ALL = {FULL: (P, I, HL), HALF: (P, I, HL), QUARTER: (P, I, HL)}
_RGB10 = {FULL: (P,), QUARTER: (P,)}
_DECODES = [("YUYV", 0, "YUYV", _ALL), ("YUYV", 0, "UYVY", _ALL), ("YUYV", 0, "PLANAR16", _ALL),
            ("YUYV", 0, "YU64", {FULL: (P,), HALF: (P, I, HL)}), ("YUYV", 0, "V210", {FULL: (P,)}),
            ("RG48", 0, "RG48", {FULL: (P,)}), ("RG48", 0, "PLANAR16", {FULL: (P,), HALF: (P,), QUARTER: (P,)}),
            ("RG48", 0, "RG30", _RGB10), ("RG48", 0, "AB10", _RGB10), ("RG48", 0, "AR10", _RGB10),
            ("RG48", 0, "R210", _RGB10), ("RG48", 0, "DPX0", _RGB10),
            ("B64A", 0, "B64A", {FULL: (P,)}), ("B64A", PKG.FRAME_ALPHA, "B64A", {FULL: (P,)}),
            ("BYR4", 0, "BYR4", {FULL: (P,)}), ("BYR5", 0, "BYR4", {FULL: (P,)}),
            ("BYR4", 0, "PLANAR16", {FULL: (P,), HALF: (P,), QUARTER: (P,)})]


def _codec(ctx, name, w, flags=0, batch=1):
    desc = PKG.FrameDesc(w, H, getattr(PKG, "PIXEL_" + name), flags)
    codec = PKG.Codec(ctx, desc, batch)
    lay = codec.layout
    return codec, desc, np.zeros((lay.frame_bytes // lay.frame_pitch, lay.frame_pitch), np.uint8)


def _forward(name, w, flags, mode, mask):
    def prepare(ctx):
        codec, desc, frame = _codec(ctx, name, w, flags)
        codec.set_interlaced(mode)
        codec.set_level_mask(mask, 7)
        quant = PKG.quant_for_quality(desc, 4, interlaced=bool(mode))
        return codec, lambda: codec.forward_host([frame], quant)
    return prepare


def _inverse(name, w, flags, out, res, mode):
    def prepare(ctx):
        codec, desc, _ = _codec(ctx, name, w, flags)
        codec.set_interlaced(mode)
        codec.set_decode_resolution(res)
        quant = PKG.quant_for_quality(desc, 4, interlaced=bool(mode))
        rw, rh = codec.decoded_size()
        frame = np.zeros((4 * rh, (8 * rw + 15) // 16 * 16), np.uint8)      # room for every output format
        coded = np.zeros(codec.layout.coded_bytes, np.uint8)
        return codec, lambda: codec.inverse_host([coded], quant, getattr(PKG, "PIXEL_" + out), [frame])
    return prepare


def _gop2(forward, mode):
    def prepare(ctx):
        codec, desc, frame = _codec(ctx, "YUYV", 384, batch=2)
        codec.set_interlaced(mode)
        gquant = PKG.gop2_quant_for_quality(desc, 4, bool(mode))
        if forward:
            return codec, lambda: codec.gop2_forward_host(frame, frame, gquant)
        coded = codec.gop2_forward_host(frame, frame, gquant)
        return codec, lambda: codec.gop2_inverse_host(coded, gquant, PKG.PIXEL_YUYV, frame.shape)
    return prepare


def _level(forward, prescale):
    plane = np.zeros((64, 100), np.int16)       # 100 wide: ragged plane and band widths
    if forward:
        return lambda ctx: (None, lambda: ctx.level_forward(plane, prescale, [1, 1, 1, 1]))
    bands = [np.zeros((32, 50), np.int16) for _ in range(4)]
    return lambda ctx: (None, lambda: ctx.level_inverse(bands, prescale, [1, 1, 1, 1]))


def _temporal(forward):
    a = np.zeros((32, 64), np.int16)
    return lambda ctx: (None, (lambda: ctx.temporal_forward(a, a)) if forward else (lambda: ctx.temporal_inverse(a, a)))


def _sparse(forward):
    def prepare(ctx):
        codec, desc, frame = _codec(ctx, "YUYV", 384)
        quant = PKG.quant_for_quality(desc, 4)
        if forward:
            return codec, lambda: codec.forward_host_sparse([frame], quant)
        sparse, _ = codec.forward_host_sparse([frame], quant)
        return codec, lambda: codec.inverse_host_sparse(sparse, quant, PKG.PIXEL_YUYV, [np.zeros((H, 768), np.uint8)])
    return prepare


def calls():
    """{id: prepare}: prepare(ctx) -> (codec or None, call); only what call() launches is counted."""
    out = {}
    for name, widths in _WIDTHS.items():
        for w in widths:
            for flags in ((0, PKG.FRAME_ALPHA) if name in ("B64A", "RG64") else (0,)):
                for mode in ((P, I) if name in _422 else (P,)):
                    for mask in (1, 7):
                        out[f"fwd-{name}-{w}-f{flags}-m{mode}-mask{mask}"] = _forward(name, w, flags, mode, mask)
    for name, flags, o, res_modes in _DECODES:
        for w in _WIDTHS[name]:
            for res, modes in res_modes.items():
                for mode in modes:
                    out[f"inv-{name}-{w}-f{flags}-{o}-r{res}-m{mode}"] = _inverse(name, w, flags, o, res, mode)
    for forward in (True, False):
        d = "fwd" if forward else "inv"
        for mode in (P, I):
            out[f"gop2-{d}-m{mode}"] = _gop2(forward, mode)
        for prescale in (0, 2):
            out[f"level-{d}-p{prescale}"] = _level(forward, prescale)
        out[f"temporal-{d}"] = _temporal(forward)
        out[f"sparse-{d}"] = _sparse(forward)
    return out


def traced(ctx, call, tries=3):
    """(kernel_launches delta, [(name, grid, block, shared memory)] of the kernels in a trace of call()).  A trace with
    no kernel at all is taken again: now and then the profiler loses a whole session (once in a full GPU suite run on an
    H100, for a call whose every other trace held its three kernels)."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(tries):
        ctx.synchronize()
        before = ctx.stats()["kernel_launches"]
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            call()
            ctx.synchronize()
        delta = ctx.stats()["kernel_launches"] - before
        with tempfile.TemporaryDirectory() as d:
            path = os.path.join(d, "trace.json")
            prof.export_chrome_trace(path)
            with open(path) as f:
                events = json.load(f)["traceEvents"]
        kernels = sorted((e for e in events if e.get("cat") == "kernel"), key=lambda e: e["ts"])
        if kernels:
            break
    return delta, [(e["name"], e["args"]["grid"], e["args"]["block"], e["args"]["shared memory"]) for e in kernels]


CALLS = calls()


def test_profiler_sees_library_kernels(ctx):
    """The library links cudart statically: the trace must still record its kernels, or the counts below prove nothing."""
    a = np.zeros((32, 64), np.int16)
    delta, kernels = traced(ctx, lambda: ctx.temporal_forward(a, a))
    assert delta == 1 and len(kernels) == 1 and "k_temporal_fwd" in kernels[0][0], kernels


@pytest.mark.parametrize("call_id", list(CALLS))
def test_counter_equals_traced_kernels(ctx, call_id):
    codec, call = CALLS[call_id](ctx)
    try:
        delta, kernels = traced(ctx, call)
    finally:
        if codec is not None:
            codec.close()
    assert kernels, "no kernel in the trace"
    assert delta == len(kernels), [k[0] for k in kernels]
