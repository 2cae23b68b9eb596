"""The 16-bit entries (include/bitnetmcu_b200.h section 11), the float top-k and scaling-only entries, and the padded window
entries (section 13) on batches and stacks whose byte offsets pass 2^31 and 2^32.

Batches are periodic, as in test_large_batches.py (tests/support.py: U unique rows, row i of a batch unique row i mod U).  The
unique rows are float16 and bfloat16 conversions of support.scattered_edge_images, so all-zero rows, rows below the 1e-5 floor,
exact .5 ties and rows with a pixel past float16's range (infinite in float16: the row scales to zeros) recur all through a batch.
A case's expected rows are the same entry on the U unique rows, pinned in the same test to the oracle (the C engine, on
restate.scale_images of the rows widened exactly with torch's .float()), to restate.emulate (the emulator) or to a stable sort of
either's logits (top-k), then tiled and compared on the device.  With 256-element rows a 16-bit batch passes 2^31 bytes at 4 M
rows and 2^32 at 8 M; a wrapped 32-bit offset would displace a read by 2^31 / 512 rows, and test_a_wrapped_offset_shows checks
on the CPU that the expected result there differs for most rows.  Every output buffer holds a sentinel past row n; the input is
checked unchanged.

Every engine case names, from its BNM_VERBOSE route line, the kernel it covers: fc_chain_h16_kernel, fc_emul_h16_kernel and
fc_engines_h16_kernel on FC 4bitsym-64, the 16-bit scaling kernel k_quantize_images<float16 / bfloat16> on every other model and
on the top-k entries, k_quantize_windows under a padded entry's name.  bnm_quantize_images_device(_f16) is that scaling kernel
called directly, with no model to print a line.

A 16-bit call on a model with 16-element rows takes the one-kernel form too (restate.plan_of: rows of at most 256 elements, at
most 16 classes), so 2^28 + 77 such rows run as two launches of fc_chain_h16_kernel, counted with torch.profiler in a process of
its own (a later profiler session in one process can miss activities).

Padded stacks: two planes whose second starts past 4 GiB (past 2^31 elements for 16-bit planes), padded on all four sides so
that the CTAs whose band reaches into the border take the padded band load; each padded entry equals its unpadded float32 sibling
on F.pad of the stack, and the border windows of the far plane equal the oracle and restate.emulate on np.pad of that plane.
Three 4096 x 4096 planes padded by 7 + 8 put the top-16 classes and scores past 2^31 bytes.

Each case states the device memory it needs, skips with that figure when the GPU has less free, and prints its n, peak device
memory and wall time."""
import functools
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import ROOT, load_model
from restate import emulate, plan_of, scale_images
from support import (SENTINEL_I32, SPARE, U, Case, GiB, Spec, check_input, check_tiled, check_wrapped_offsets, lib,  # noqa: F401
                     need, outputs, periodic, random_fc, scattered_edge_images, top_k, verbose_engine, views, want_on_device)
# (lib: a fixture)

FORMATS = ["float16", "bfloat16"]
N23, N24 = ((1 << b) + 77 for b in (23, 24))
K_FUSED_PASS = 1 << 28          # images per fused FC launch (kFusedPass, capi.cu)

MODELS = {
    "fc": lambda: load_model("fc"),                                 # 4bitsym-64: the one-kernel 16-bit forms
    "head47": lambda: random_fc(16, (256, 64, 47), 47),             # 47 classes: no float-input form, the scaling kernel
    "binary160": lambda: load_model("binary160"),                   # <192,1>: no float-input form
    "cnn_48": lambda: load_model("cnn_48"),                         # the CNN front-end behind the scaling pass
    "fc16": lambda: random_fc(16, (16, 16, 10), 16),                # 16-element rows
}
K = {"head47": 16, "fc": 10}    # top-k: 16, or the class count


@functools.lru_cache(maxsize=None)
def model(name):
    return MODELS[name]()


# ---- the unique rows and what every entry gives on them (CPU) ---------------------------------------------------------------

@functools.lru_cache(maxsize=None)
def rows(name, fmt):
    """the U unique rows of model `name` in fmt: float32 NumPy, or a CPU torch tensor of float16 / bfloat16"""
    import torch
    x = scattered_edge_images(U, model(name).img_bytes, seed=len(name) * 13 + 5)
    return x if fmt == "float32" else torch.from_numpy(x).to(getattr(torch, fmt))


def widened(name, fmt):
    """the unique rows as float32, widened exactly"""
    r = rows(name, fmt)
    return r if fmt == "float32" else r.float().numpy()


_EXPECTED = {}


def expected(oracle, kind, name, fmt):
    """what entry `kind` gives on the unique rows of model `name` in fmt: {output: NumPy [U, ...]}"""
    key = (kind, name, fmt)
    if key not in _EXPECTED:
        m = model(name)
        if kind == "c":
            lo, la = oracle.infer(m, scale_images(widened(name, fmt)))
            r = {"logits": lo, "labels": la}
        elif kind == "emul":
            lo = emulate(m, widened(name, fmt))
            r = {"logits": lo, "labels": np.argmax(lo, axis=1).astype(np.uint32)}
        elif kind == "engines":
            r = {"labels_c": expected(oracle, "c", name, fmt)["labels"], "labels_py": expected(oracle, "emul", name, fmt)["labels"]}
        elif kind in ("topk", "emul_topk"):
            cls, sc = top_k(expected(oracle, "c" if kind == "topk" else "emul", name, fmt)["logits"], K[name])
            r = {"classes": cls, "scores": sc}
        elif kind == "quant":
            r = {"q": scale_images(widened(name, fmt))}
        _EXPECTED[key] = r
    return _EXPECTED[key]


def _specs():
    """case -> (format, Spec); 256-element rows: 512 bytes in 16-bit, 1024 in float32"""
    out = {}
    two = ("logits", "labels")
    for fmt in FORMATS:
        specs = {
            f"c fc {fmt}": Spec("c", "fc", N23, 512, two),
            f"c fc labels only {fmt}": Spec("c", "fc", N23, 512, ("labels",)),
            f"emulator fc {fmt}": Spec("emul", "fc", N23, 512, two),
            f"engines fc {fmt}": Spec("engines", "fc", N23, 512, ("labels_c", "labels_py")),
            f"emulator head47 {fmt}": Spec("emul", "head47", N23, 512, two),       # float64 logits past 2^31 bytes
            f"c binary160 {fmt}": Spec("c", "binary160", N23, 512, two),
            f"c cnn_48 {fmt}": Spec("c", "cnn_48", N23, 512, two),
            f"topk head47 {fmt}": Spec("topk", "head47", N24, 512, ("classes", "scores")),
            f"emulator topk head47 {fmt}": Spec("emul_topk", "head47", N24, 512, ("classes", "scores")),   # scores past 2^31
            f"topk fc {fmt}": Spec("topk", "fc", N24, 512, ("classes", "scores")),
            f"emulator topk fc {fmt}": Spec("emul_topk", "fc", N24, 512, ("classes", "scores")),
            f"quantize {fmt}": Spec("quant", "fc", N24, 512, ("q",)),               # int8 rows past 2^32 bytes
        }
        out.update({k: (fmt, s) for k, s in specs.items()})
    out.update({
        "topk head47 float32": ("float32", Spec("topk", "head47", N23, 1024, ("classes", "scores"))),
        "emulator topk head47 float32": ("float32", Spec("emul_topk", "head47", N23, 1024, ("classes", "scores"))),
        "quantize float32": ("float32", Spec("quant", "fc", N23, 1024, ("q",))),   # int8 rows past 2^31 bytes, input past 2^33
    })
    return out


SPECS = _specs()
# the split of a 16-bit batch of 16-element rows into fused launches
SPLIT = Spec("c", "fc16", K_FUSED_PASS + 77, 32, ("labels",))


# ---- CPU ----------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("case", list(SPECS))
def test_a_wrapped_offset_shows(oracle, case):
    """for every read and write whose offsets pass a wrap W (2^31 or 2^32 bytes), the result a read or write displaced by W
    would give differs from the expected one for most rows"""
    fmt, s = SPECS[case]
    check_wrapped_offsets(case, s, expected(oracle, s.kind, s.name, fmt))


def test_wrapped_offset_shows_on_the_split(oracle):
    check_wrapped_offsets("split fc16", SPLIT, expected(oracle, "c", "fc16", "float16"))


def test_unique_rows_hold_the_scaling_edges():
    """the unique rows hold all-zero rows (under the 1e-5 floor: they scale to zeros) in every format, and in 16-bit rows with
    an exact .5 product (a round-half-even tie) and, in float16 only, rows with an infinite pixel, which scale to zeros"""
    import torch
    for fmt in FORMATS + ["float32"]:
        w = widened("fc", fmt)
        q = scale_images(w)
        zero = ~w.any(axis=1)
        assert zero.sum() > U // 20 and not q[zero].any(), fmt
        inf = ~np.isfinite(w).all(axis=1)
        assert (inf.sum() > U // 20) == (fmt == "float16") and not q[inf].any(), fmt
        with np.errstate(invalid="ignore", over="ignore"):
            y = w * (np.float32(127.0) / np.maximum(np.abs(w).max(axis=1, keepdims=True), np.float32(1e-5)))
            ties = (np.abs(y - np.trunc(y)) == 0.5).any(axis=1)
        assert fmt == "float32" or ties.sum() > 50, (fmt, ties.sum())
    assert torch.equal(rows("fc", "float16").float(), torch.from_numpy(widened("fc", "float16")))


def test_16bit_form_takes_16_element_rows():
    """the 16-bit one-kernel form takes a model of 16-element rows, so a batch of such rows is split into launches of 2^28
    (kFusedPass) by that form's route"""
    plan = plan_of(model("fc16"))
    assert plan.forms["float16"].row == "fc_chain_h16_kernel<64,1,16bit>", plan
    assert SPLIT.n > K_FUSED_PASS and SPLIT.n * SPLIT.in_bytes > 1 << 33


# ---- GPU: the entries on periodic batches --------------------------------------------------------------------------------------

def _engine(name):
    from bitnetmcu_b200.engine import Engine
    return Engine(model(name), device=0)


ENTRY = {("c", False): "bnm_infer_batch_device_f16", ("emul", False): "bnm_emulate_batch_device_f16",
         ("engines", False): "bnm_compare_engines_device_f16", ("topk", False): "bnm_infer_topk_device_f16",
         ("emul_topk", False): "bnm_emulate_topk_device_f16", ("topk", True): "bnm_infer_topk_device_f32",
         ("emul_topk", True): "bnm_emulate_topk_device"}
ONE_KERNEL = {("c", "fc"): "fc_chain_h16_kernel<64,1,16bit>", ("c", "fc16"): "fc_chain_h16_kernel<64,1,16bit>",
              ("emul", "fc"): "fc_emul_h16_kernel<64,1,16bit,emul>", ("engines", "fc"): "fc_engines_h16_kernel<64,1,16bit,engines>"}
AFTER_SCALING = {("emul", "head47"): "fc_emul_i8_kernel<64,1,emul>", ("c", "binary160"): "fc_chain_kernel<192,1>",
                 ("c", "cnn_48"): "k_cnn_frontend16", "topk": "fc_topk_kernel<64,1,topk>", "emul_topk": "fc_topk_kernel<64,1,emul,topk>"}


def route_line(kind, name, fmt):
    """what the BNM_VERBOSE route line of the call holds: the entry, then the one-kernel form, or the scaling kernel of fmt and
    what runs on its rows"""
    topk = kind in ("topk", "emul_topk")
    head = ("topk route: " if topk else "16-bit route: ") + ENTRY[(kind, fmt == "float32")] + ": "
    if (kind, name) in ONE_KERNEL:
        return head + ONE_KERNEL[(kind, name)]
    scale = "k_quantize_images + " if fmt == "float32" else f"k_quantize_images<{fmt}> + "
    return head + scale + AFTER_SCALING[kind if topk else (kind, name)]


def run(e, kind, x, o, k=None):
    """the device entry of `kind` on images x into the output views o"""
    from bitnetmcu_b200.engine import quantize_images_device
    if kind == "c":
        e.infer_device_f32(x, o.get("logits"), o.get("labels"))
    elif kind == "emul":
        e.inference_quantized_device(x, o.get("logits"), o.get("labels"))
    elif kind == "engines":
        e.compare_engines_device(x, labels_c=o["labels_c"], labels_py=o["labels_py"])
    elif kind == "topk":
        e.topk_device_f32(x, k, o["classes"], o["scores"])
    elif kind == "emul_topk":
        e.emulate_topk_device(x, k, o["classes"], o["scores"])
    elif kind == "quant":
        quantize_images_device(x, o["q"])


def route_lines(capfd):
    import torch
    torch.cuda.synchronize()
    return [l for l in capfd.readouterr().err.splitlines() if "route: " in l]


def entry_case(oracle, capfd, monkeypatch, case):
    """case `case` of SPECS: the small call on the unique rows pinned to the reference and naming its route, the periodic batch
    of n rows against it tiled, the sentinels, the input"""
    import torch
    fmt, s = SPECS[case]
    res = expected(oracle, s.kind, s.name, fmt)
    with Case(case, s.n, need(s, res)) as c:
        e = None
        if s.kind != "quant":
            e, _ = verbose_engine(capfd, monkeypatch, lambda: c.engine(lambda: _engine(s.name)))
        u = rows(s.name, fmt)
        small = outputs(res, s.outputs, U)
        capfd.readouterr()
        run(e, s.kind, (u if fmt != "float32" else torch.from_numpy(u)).cuda(), views(small, U), K.get(s.name))
        lines = route_lines(capfd)
        if e is not None:
            want = route_line(s.kind, s.name, fmt)
            assert len(lines) == 1 and want in lines[0], (case, want, lines)
        want = want_on_device(small, res, case)
        x = periodic(u, s.n)
        got = outputs(res, s.outputs, s.n)
        run(e, s.kind, x, views(got, s.n), K.get(s.name))
        torch.cuda.synchronize()
        check_tiled(got, want, s.n, s.uid, case)
        check_input(x, u, case)
        del x, got, small, want


def _cases(*kinds, fmts=tuple(FORMATS)):
    return [c for c, (fmt, s) in SPECS.items() if s.kind in kinds and fmt in fmts]


@pytest.mark.gpu
@pytest.mark.parametrize("case", [c for c in _cases("c", "emul", "engines") if " fc " in c])
def test_one_kernel_forms(lib, oracle, capfd, monkeypatch, case):
    """fc_chain_h16_kernel (logits and labels, labels only), fc_emul_h16_kernel and fc_engines_h16_kernel on 2^23 + 77 rows:
    the quantiser warps' bulk loads from src + row * elems past 4 GiB"""
    entry_case(oracle, capfd, monkeypatch, case)


@pytest.mark.gpu
@pytest.mark.parametrize("case", [c for c in _cases("c", "emul") if " fc " not in c])
def test_scaling_kernel_route(lib, oracle, capfd, monkeypatch, case):
    """k_quantize_images<float16 / bfloat16> into per-pass scratch, input past 4 GiB: the emulator on head47 (float64 logits past
    2^31 bytes), the C engine on binary160 and on cnn_48 (its front-end behind the scaling pass)"""
    entry_case(oracle, capfd, monkeypatch, case)


@pytest.mark.gpu
@pytest.mark.parametrize("case", _cases("topk", "emul_topk", fmts=("float16", "bfloat16", "float32")))
def test_topk(lib, oracle, capfd, monkeypatch, case):
    """classes and scores of the C engine and the emulator: 16-bit rows past 8 GiB (the emulator's top-16 scores past 2^31
    bytes), float32 rows past 8 GiB"""
    entry_case(oracle, capfd, monkeypatch, case)


@pytest.mark.gpu
@pytest.mark.parametrize("case", _cases("quant", fmts=("float16", "bfloat16", "float32")))
def test_quantize_images(lib, oracle, capfd, monkeypatch, case):
    """bnm_quantize_images_device(_f16): 16-bit rows into int8 rows past 2^32 bytes, float32 rows into int8 rows past 2^31"""
    entry_case(oracle, capfd, monkeypatch, case)


def split_run(expected_path):
    """the split case, in a process of its own: 16-element float16 rows, 2^28 + 77 of them, labels only, against the small
    call pinned by the caller (expected_path: its labels); prints the case line, then {"launches": fc_chain_h16_kernel launches
    of the large call} as JSON, or {"skip": why}"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    s = SPLIT
    res = {"labels": np.load(expected_path)}
    try:
        with Case("split fc16 labels only float16", s.n, need(s, res)) as c:
            e = c.engine(lambda: _engine("fc16"))
            u = rows("fc16", "float16")
            small = outputs(res, s.outputs, U)
            run(e, "c", u.cuda(), views(small, U))
            torch.cuda.synchronize()
            want = want_on_device(small, res, "fc16")
            x = periodic(u, s.n)
            got = outputs(res, s.outputs, s.n)
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                run(e, "c", x, views(got, s.n))
                torch.cuda.synchronize()
            names = [ev.name for ev in prof.events() if ev.device_type == torch.autograd.DeviceType.CUDA]
            check_tiled(got, want, s.n, s.uid, "split")
            check_input(x, u, "split")
            del x, got
    except pytest.skip.Exception as why:
        print(json.dumps({"skip": str(why)}))
        return
    print(json.dumps({"launches": sum("fc_chain_h16_kernel" in n for n in names)}))


@pytest.mark.gpu
def test_16bit_batch_splits_into_launches(lib, oracle, tmp_path):
    """2^28 + 77 float16 rows of 16 elements, labels only: two launches of fc_chain_h16_kernel (the route line names it), which
    equal the tiled small call, sentinels and input intact"""
    import torch
    path = str(tmp_path / "labels.npy")
    np.save(path, expected(oracle, "c", "fc16", "float16")["labels"])
    torch.cuda.empty_cache()
    script = f"""
import sys
sys.path[:0] = [{ROOT!r}, {os.path.join(ROOT, "tests")!r}]
from test_large_batches_16bit import split_run
split_run({path!r})
"""
    env = dict(os.environ, BNM_VERBOSE="1")
    done = subprocess.run([sys.executable, "-c", script], capture_output=True, text=True, cwd=ROOT, env=env, timeout=1200)
    assert done.returncode == 0, done.stderr[-3000:]
    out = done.stdout.strip().splitlines()
    print("\n".join(out[:-1]))
    r = json.loads(out[-1])
    if "skip" in r:
        pytest.skip(r["skip"])
    assert route_line("c", "fc16", "float16") in done.stderr, done.stderr[-3000:]
    assert r["launches"] == 2, r


# ---- GPU: padded stacks ---------------------------------------------------------------------------------------------------------

PAD_MODES = {"constant": "constant", "replicate": "edge", "reflect": "reflect"}   # torch's names -> NumPy's
PAD = (7, 8, 15, 1)             # left, right, top, bottom
ENTRIES = ["scan", "scan_topk", "emulate", "emulate_topk"]
STEMS = {"scan": "bnm_scan_windows", "scan_topk": "bnm_scan_windows_topk", "emulate": "bnm_emulate_windows",
         "emulate_topk": "bnm_emulate_windows_topk"}


def page_pixels(planes, h, w, seed):
    """normal pixels at a scale per row, a dark left margin and a bright bottom row: float32 [planes, h, w]"""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((planes, h, w), dtype=np.float32) * (10.0 ** rng.uniform(-2, 2, (planes, h, 1))).astype(np.float32)
    x[:, :, :3] *= np.float32(1e-3)
    x[:, -1, :] = np.float32(40.0)
    return x


def run_windows(e, entry, pages, stride, k, padding=None, mode="constant", value=0.0):
    """the window entry on a CUDA stack -> its two outputs as CUDA tensors [windows, ...]: (logits, labels) or (classes, scores)"""
    import torch
    from bitnetmcu_b200.engine import window_grid
    grid = (pages.shape[0],) + window_grid(pages.shape[1], pages.shape[2], stride, padding)
    emul, topk = entry.startswith("emulate"), entry.endswith("topk")
    kw = {} if padding is None else {"padding": padding, "pad_mode": mode, "pad_value": value}
    f = lambda shape, dt: torch.full(grid + shape, SENTINEL_I32, dtype=dt, device="cuda")
    sdt = torch.float64 if emul else torch.int32
    if topk:
        a, b = f((k,), torch.int32), f((k,), sdt)
        (e.emulate_windows_topk_device if emul else e.scan_windows_topk_device)(pages, stride, k, a, b, **kw)
    else:
        a, b = f((e.n_classes,), sdt), f((), torch.int32)
        (e.emulate_windows_device if emul else e.scan_windows_device)(pages, stride, a, b, **kw)
    torch.cuda.synchronize()
    n = int(np.prod(grid))
    return a.reshape(n, -1), b.reshape(n, -1)


def padded_copy(pages, pad, mode, value):
    """F.pad(pages.float(), pad, mode, value): what a caller passes the unpadded sibling, in a float32 stack whose rows are
    16-byte multiples apart"""
    import torch
    import torch.nn.functional as F
    x = pages.float()
    x = F.pad(x, pad, mode="constant", value=value) if mode == "constant" else F.pad(x, pad, mode=mode)
    p, h, w = x.shape
    out = torch.empty((p, h, (w + 3) // 4 * 4), dtype=torch.float32, device="cuda")[:, :, :w]
    out.copy_(x)
    return out


def first_bad(got, want):
    """the first rows of got that differ from want"""
    import torch
    return torch.nonzero((got != want).reshape(got.shape[0], -1).any(dim=1))[:6, 0].tolist()


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["float32"] + FORMATS)
def test_padded_stack_past_4_gib(lib, oracle, capfd, monkeypatch, fmt):
    """two 40 x 64 planes, the second past 4 GiB (16-bit: past 2^31 elements), padded 7 / 8 / 15 / 1 in every mode at strides 1
    and 4: every padded entry (logits and labels, top-k classes and scores, of the C engine and the emulator) equals its float32
    sibling on F.pad of the stack, names k_quantize_windows under its padded name, and the border windows of the far plane equal
    the oracle and restate.emulate on np.pad of that plane"""
    import torch
    dt = getattr(torch, fmt)
    plane_pitch = ((1 << 30) if fmt == "float32" else (1 << 31)) + 256     # elements
    h, w = 40, 64
    left, right, top, bottom = PAD
    with Case(f"padded stack {fmt}, two 40 x 64 planes (pixels)", 2 * h * w, plane_pitch * dt.itemsize + GiB) as c:
        e, _ = verbose_engine(capfd, monkeypatch, lambda: c.engine(lambda: _engine("fc")))
        buf = torch.full((plane_pitch + h * w,), float("nan"), dtype=dt, device="cuda")
        pages = buf.as_strided((2, h, w), (plane_pitch, w, 1))
        pages.copy_(torch.from_numpy(page_pixels(2, h, w, seed=len(fmt))).to(dt))
        assert pages[1].data_ptr() - pages.data_ptr() > 4 << 30 and (fmt == "float32" or plane_pitch > 1 << 31)
        far = pages[1].float().cpu().numpy()
        scale = "k_quantize_windows + " if fmt == "float32" else f"k_quantize_windows<{fmt}> + "
        for mode in PAD_MODES:
            value = -1.5
            sibling_pages = padded_copy(pages, PAD, mode, value)
            kw = {"constant_values": np.float32(value)} if mode == "constant" else {}
            far_padded = np.pad(far, ((top, bottom), (left, right)), mode=PAD_MODES[mode], **kw)
            for stride in (1, 4):
                oh, ow = (h + top + bottom - 16) // stride + 1, (w + left + right - 16) // stride + 1
                ring = sorted({(r, cc) for r in range(oh) for cc in range(ow) if r in (0, oh - 1) or cc in (0, ow - 1)})
                ids = np.array([oh * ow + r * ow + cc for r, cc in ring])     # the far plane's border windows
                wins = np.stack([far_padded[r * stride:r * stride + 16, cc * stride:cc * stride + 16].reshape(256) for r, cc in ring])
                for entry in ENTRIES:
                    what = (fmt, mode, stride, entry)
                    capfd.readouterr()
                    got = run_windows(e, entry, pages, stride, 5, PAD, mode, value)
                    lines = route_lines(capfd)
                    name = STEMS[entry] + "_padded_device" + ("" if fmt == "float32" else "_f16")
                    assert len(lines) == 1 and f"windows route: {name}: {scale}" in lines[0], (what, lines)
                    want = run_windows(e, entry, sibling_pages, stride, 5)
                    for g, wt, o in zip(got, want, ("first", "second")):
                        assert g.shape == wt.shape and bool((g == wt).all()), (what, o, "windows differ", first_bad(g, wt))
                    if entry == "scan":
                        lo, la = oracle.infer(e.model, scale_images(wins))
                        assert np.array_equal(got[0][ids].cpu().numpy(), lo), (what, "border logits")
                        assert np.array_equal(got[1][ids, 0].cpu().numpy().astype(np.uint32), la), (what, "border labels")
                    elif entry == "emulate":
                        lo = emulate(e.model, wins)
                        assert np.array_equal(got[0][ids].cpu().numpy(), lo), (what, "border emulator logits")
        del pages, buf


@pytest.mark.gpu
def test_padded_topk_outputs_past_2_31(lib, capfd, monkeypatch):
    """three 4096 x 4096 planes padded 7 + 8 on every side (reflect) at stride 1: the top-16 classes and scores of head47 pass
    2^31 bytes (3.2 GB each), and equal the unpadded sibling on each plane's padded copy; nothing is written past them"""
    import torch
    n_p, side, k = 3, 4096, 16
    per = side * side
    n = n_p * per
    res = {"classes": np.zeros((1, k), np.int32), "scores": np.zeros((1, k), np.int32)}
    assert n * k * 4 > 1 << 31
    with Case("padded topk head47 4096 x 4096 x 3", n, 2 * (n + SPARE) * k * 4 + per * k * 8 + 2 * GiB) as c:
        e, _ = verbose_engine(capfd, monkeypatch, lambda: c.engine(lambda: _engine("head47")))
        g = torch.Generator(device="cuda").manual_seed(47)
        pages = torch.randn((n_p, side, side), generator=g, device="cuda")
        pages[:, :, :40] *= 1e-3
        got = outputs(res, ("classes", "scores"), n)
        v = views(got, n, (n_p, side, side))
        capfd.readouterr()
        e.scan_windows_topk_device(pages, 1, k, v["classes"], v["scores"], padding=(7, 8, 7, 8), pad_mode="reflect")
        lines = route_lines(capfd)
        want = "windows route: bnm_scan_windows_topk_padded_device: k_quantize_windows + fc_topk_kernel"
        assert len(lines) == 1 and want in lines[0], lines
        for p in range(n_p):
            sib = padded_copy(pages[p:p + 1], (7, 8, 7, 8), "reflect", 0.0)
            cls, sc = run_windows(e, "scan_topk", sib, 1, k)
            for o, wt in (("classes", cls), ("scores", sc)):
                t = got[o][p * per:(p + 1) * per]
                for s in range(0, per, 1 << 22):
                    bad = first_bad(t[s:s + (1 << 22)], wt[s:s + (1 << 22)])
                    assert not bad, (o, f"plane {p}", "windows wrong, first", [p * per + s + b for b in bad],
                                     "byte offsets", [(p * per + s + b) * k * 4 for b in bad])
            del sib, cls, sc
        for o, t in got.items():
            assert bool((t[n:] == SENTINEL_I32).all()), (o, "written past the last window")
        del pages, got, v
