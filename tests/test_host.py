"""CPU tests of the host side: C-ABI library loads and exports every declared symbol, the module mirror
strict-loads reference-format checkpoints, window arithmetic, loud failure without CUDA."""
import ctypes
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_builds_and_exports_every_declared_symbol():
    from marconet_b200 import _lib, build
    build.build()
    lib = _lib.load()
    header = open(os.path.join(ROOT, "include", "marconet_b200.h")).read()
    declared = set(re.findall(r"\b(mn_[a-z0-9_]+)\s*\(", header))
    declared -= {"mn_status", "mn_act", "mn_precision"}
    assert declared, "no declarations parsed"
    raw = ctypes.CDLL(_lib.LIB_PATH)
    for name in sorted(declared):
        assert hasattr(raw, name), f"{name} declared in include/marconet_b200.h but not exported"
        assert name in _lib.SYMBOLS, f"{name} has no ctypes binding"
    assert lib.mn_version() >= 100


def test_ctypes_signatures_match_the_header_prototypes():
    """Every prototype of include/marconet_b200.h against its ctypes binding: argument count and argument class (pointer /
    int / long long / float / double) and the return type -- a wrong binding would otherwise only show up on the GPU box."""
    from marconet_b200 import _lib
    header = open(os.path.join(ROOT, "include", "marconet_b200.h")).read()
    header = re.sub(r"/\*.*?\*/", "", header, flags=re.S)
    protos = re.findall(r"(?m)^\s*(const char\s*\*|int64_t|int)\s+(mn_[a-z0-9_]+)\s*\(([^;{]*?)\)\s*;", header)
    assert len(protos) >= 30

    def klass(decl):
        decl = decl.strip()
        if decl == "void":
            return None
        if "*" in decl:
            return "ptr"
        if re.search(r"\blong long\b|\bint64_t\b", decl):
            return "i64"
        if re.search(r"\bdouble\b", decl):
            return "f64"
        if re.search(r"\bfloat\b", decl):
            return "f32"
        if re.search(r"\b(int|int32_t|unsigned)\b", decl):
            return "i32"
        raise AssertionError(f"unparsed parameter {decl!r}")

    def cklass(t):
        if t in (ctypes.c_void_p, ctypes.c_char_p) or hasattr(t, "contents") or (isinstance(t, type) and issubclass(t, ctypes._Pointer)):
            return "ptr"
        return {ctypes.c_int: "i32", ctypes.c_int32: "i32", ctypes.c_longlong: "i64", ctypes.c_int64: "i64", ctypes.c_float: "f32",
                ctypes.c_double: "f64"}[t]

    seen = set()
    for ret, name, params in protos:
        want = [k for k in (klass(p) for p in params.split(",")) if k is not None]
        restype, argtypes = _lib.SYMBOLS[name]
        assert [cklass(t) for t in argtypes] == want, f"{name}: header {want} vs ctypes {[cklass(t) for t in argtypes]}"
        assert restype is {"int": ctypes.c_int, "int64_t": ctypes.c_int64}.get(ret, ctypes.c_char_p), name
        seen.add(name)
    assert seen == set(_lib.SYMBOLS), sorted(set(_lib.SYMBOLS) ^ seen)


def test_conv_params_struct_matches_header_field_order():
    from marconet_b200 import _lib
    header = open(os.path.join(ROOT, "include", "marconet_b200.h")).read()
    body = header.split("typedef struct {", 1)[1].split("} mn_conv_params;")[0]
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = []
    for decl in body.split(";"):
        decl = decl.strip()
        if not decl:
            continue
        parts = [p.strip() for p in decl.split(",")]
        names.append(re.findall(r"[A-Za-z_0-9]+$", parts[0])[0])
        names += [re.findall(r"[A-Za-z_0-9]+$", p)[0] for p in parts[1:]]
    assert names == [f[0] for f in _lib.ConvParams._fields_]


def test_strict_load_and_param_counts(checkpoints):
    from marconet_b200.models import networks
    want = {"tspgan": 27970194, "encoder": 43062275, "sr": 16865923}       # banner of test_sr.py:59-61
    for key, cls in (("tspgan", networks.TSPGAN), ("encoder", networks.TextContextEncoderV2), ("sr", networks.TSPSRNet)):
        m = cls()
        m.load_state_dict(checkpoints[key], strict=True)
        assert list(m.state_dict().keys()) == list(checkpoints[key].keys())
        assert sum(p.numel() for p in m.parameters()) == want[key]
        for k, v in m.state_dict().items():
            assert v.shape == checkpoints[key][k].shape


def test_helper_classes_importable_under_reference_names():
    import importlib
    import sys
    sys.path.insert(0, os.path.join(ROOT, "dropin"))
    try:
        for name in [m for m in sys.modules if m == "models" or m.startswith("models.")]:
            del sys.modules[name]
        nets = importlib.import_module("models.networks")
        importlib.import_module("models.ocr")
        for cls in ("TSPGAN", "TextGenerator", "TSPSRNet", "TextContextEncoderV2", "StyledConv", "ModulatedConv2d", "ToRGB",
                    "EqualLinear", "SelectText", "PixelNorm", "ResTextBlockV2"):
            assert hasattr(nets, cls), cls
    finally:
        sys.path.remove(os.path.join(ROOT, "dropin"))
        for name in [m for m in sys.modules if m == "models" or m.startswith("models.")]:
            del sys.modules[name]


def test_cpu_inputs_fail_loudly(checkpoints):
    from marconet_b200.models import networks
    m = networks.TSPGAN()
    with pytest.raises(RuntimeError, match="CUDA"):
        m(torch.randn(1, 512), torch.zeros(1, 1, dtype=torch.long), None)
    with pytest.raises(RuntimeError, match="CUDA"):
        networks.TextContextEncoderV2()(torch.randn(1, 3, 32, 512))


def test_char_windows_ownership_last_writer_wins():
    from marconet_b200.models.networks import char_windows
    locs = torch.tensor([[100.2 / 512, 0.03, 110.9 / 512, 0.03, 3.0 / 512, 0.03, 509.0 / 512, 0.03]])
    wins, valid, owner = char_windows(locs, [4], 512, 16)
    assert wins == [(0, 84, 116, 0), (0, 94, 126, 0), (0, 0, 19, 7), (0, 493, 512, 7)]
    assert valid == [32, 32, 19, 19]
    assert owner[0][90] == 0 and owner[0][100] == 1 and owner[0][120] == 1 and owner[0][5] == 2 and owner[0][200] == -1
    with pytest.raises(RuntimeError):
        char_windows(torch.tensor([[-0.2, 0.0]]), [1], 512, 16)


def test_char_windows_match_a_literal_restatement_on_random_boxes():
    """Window integers (INT parity, SURVEY 8a a12): the host function against the reference's statements executed literally with
    0-dim torch tensors (networks.py:426-441 for the 32-row level, :460-474 for the 64-row level), on random and adversarial
    centres (products that land within one ulp of an integer, the clipped ends)."""
    import torch
    from marconet_b200.models.networks import char_windows
    g = torch.Generator().manual_seed(123)
    for width, half in ((512, 16), (1024, 32)):
        centres = [torch.rand(64, generator=g)]
        k = torch.arange(1, 65, dtype=torch.float32) * 7
        centres += [k / width, torch.nextafter(k / width, torch.tensor(0.0)), torch.nextafter(k / width, torch.tensor(2.0))]
        centres.append(torch.tensor([0.0, 1.0, 15.999 / width, 16.0 / width, (width - 16.0) / width, (width - 15.999) / width] + [0.5] * 58))
        locs = torch.zeros(len(centres), 128)
        for b, c in enumerate(centres):
            locs[b, 0::2] = c
        counts = [64] * len(centres)
        wins, valid, owner = char_windows(locs, counts, width, half)
        i = 0
        for b in range(len(centres)):
            for c in range(64):
                center = (locs[b][2 * c] * width).int()
                wd = half
                if center < wd:
                    x1 = 0
                else:
                    x1 = center - wd
                if center + wd > width:
                    x2 = width
                else:
                    x2 = center + wd
                y1 = half - torch.div(x2 - x1, 2, rounding_mode='trunc')
                assert wins[i] == (b, int(x1), int(x2), int(y1)) and valid[i] == int(x2 - x1), (width, b, c, wins[i])
                i += 1
        # ownership: the last character in program order whose window covers the column
        for b in range(len(centres)):
            expect = [-1] * width
            for c in range(64):
                _, x1, x2, _ = wins[b * 64 + c]
                for x in range(x1, x2):
                    expect[x] = b * 64 + c
            assert owner[b] == expect


def test_launch_context_is_per_thread():
    """ops.use_workspace / ops.deferred_checks are thread-local (ADVICE r1): a second host thread must not see the scratch or the
    error flag another thread installed."""
    import threading
    from marconet_b200 import ops

    class _Fake:            # stands in for a CUDA tensor: deferred_checks only validates real flags when they are not None
        pass

    seen = {}
    ready, done = threading.Event(), threading.Event()

    def other():
        ready.wait(5)
        seen["ws"] = getattr(ops._TLS, "ws_override", None)
        seen["flag"] = ops.deferred_flag()
        done.set()

    t = threading.Thread(target=other)
    t.start()
    marker = _Fake()
    with ops.use_workspace(marker):
        ops._TLS.deferred_flag = marker
        try:
            assert ops.workspace(None) is marker and ops.deferred_flag() is marker
            ready.set()
            done.wait(5)
        finally:
            ops._TLS.deferred_flag = None
    t.join()
    assert seen == {"ws": None, "flag": None}


def test_precision_plan_survives_repack_by_name():
    """ops.PLAN is keyed by layer name: a ConvWeight re-created under the same name picks its precision / input scale up again."""
    import torch
    from marconet_b200 import ops
    saved = dict(ops.PLAN)
    try:
        a = ops.ConvWeight(torch.zeros(9 * 64, 64), 9, name="test.plan_layer")
        assert (a.precision, a.x_scale) == (None, 1.0)
        a.set_plan(precision=ops.PREC_BF16X3_TC, x_scale=0.25)
        b = ops.ConvWeight(torch.zeros(9 * 64, 64), 9, name="test.plan_layer")
        assert (b.precision, b.x_scale) == (ops.PREC_BF16X3_TC, 0.25)
        assert ops.ConvWeight.from_tag(b.tag) is b
    finally:
        ops.PLAN.clear()
        ops.PLAN.update(saved)


def test_range_slots_belong_to_live_layers_and_are_reused():
    """Each live tensor-core layer has its own range-flag slot, whatever its tag: two layers whose tags are congruent modulo the
    slot count (tags only grow, every re-pack makes new layers) must not share one.  A dead layer's slot goes back to the pool."""
    import gc
    import torch
    from marconet_b200 import ops
    gc.collect()                                     # dead layers of earlier tests give their slots back now, not below
    a = ops.ConvWeight(torch.zeros(64, 64), 1, name="test.slot_a")
    ops.ConvWeight._next_tag = a.tag + ops._RANGE_SLOTS
    b = ops.ConvWeight(torch.zeros(64, 64), 1, name="test.slot_b")
    assert b.tag % ops._RANGE_SLOTS == a.tag % ops._RANGE_SLOTS
    sa, sb = a.range_slot(), b.range_slot()
    assert sa != sb and a.range_slot() == sa and 0 <= min(sa, sb) and max(sa, sb) < ops._RANGE_SLOTS
    tag_b = b.tag
    del b
    gc.collect()
    assert ops.ConvWeight.from_tag(tag_b) is None and tag_b not in ops.ConvWeight._by_tag
    free = list(ops._RANGE_POOL.free)
    assert sb in free                                # b's slot went back to the pool
    c = ops.ConvWeight(torch.zeros(64, 64), 1, name="test.slot_c")
    assert c.range_slot() == free[-1] and c.range_slot() != sa     # a released slot is reused before a new one is taken
    assert ops.ConvWeight.from_tag(a.tag) is a and a.range_slot() == sa


def test_range_slot_pool_raises_beyond_its_size():
    """More live layers than slots is an error naming the limit, not a silently shared flag; a released slot makes room again."""
    import pytest
    from marconet_b200 import ops
    pool = ops._SlotPool(3)
    got = [pool.take() for _ in range(3)]
    assert sorted(got) == [0, 1, 2]
    with pytest.raises(RuntimeError, match="more than 3 live tensor-core conv layers"):
        pool.take()
    pool.give(got[1])
    assert pool.take() == got[1]

