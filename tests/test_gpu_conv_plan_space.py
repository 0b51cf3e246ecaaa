"""The tensor-core convolution across its plan space, every output element against fp64 (oracle/conv_ref.py ``conv_ref_full``).

The module sweeps (test_gpu_conv_sweep.py) check the convolutions the three modules make, at sampled pixels and with the full
persistent grid.  Here a fixed list of geometries reaches every outcome of the planner -- both tilings, both work-item widths, tiles
of one and of several samples, split-K 1/2/4/8, one- and two-CTA clusters (with the padding CTA of an odd tile count), samples that
do not fill the last tile, both ring depths -- and each is checked:
  - at f16x3 and bf16x3, plain and with the full epilogue (bias, per-sample out_scale, residual, LReLU with gain, a second output with
    y2_scale, ragged valid_w including 1); with the fused GroupNorm input and the epilogue statistics, and with per-sample output
    pointers, where the plan honours them;
  - NaN in the input channels outside the slice, NaN in every output element before the call (each must be written, masked ones
    as 0), GUARD around the output slice and in a guard sample after it (must stay);
  - under CTA caps of 1, 5 and 7 (``ops.set_max_ctas``), where one cluster walks many work items and its A / weight mbarrier rings
    wrap across item boundaries: y and y2 bit-identical to the uncapped call (each output tile is owned by one cluster, the
    accumulation order inside an item is fixed and split-K sizes from the SM count, not the cap);
  - with programmatic dependent launch off: a chain of dependent launches at cap 1 gives the same bits as with PDL on and as with a
    synchronisation after every call;
  - split-K under workspaces too small for the planned split, and the geometries the planner must refuse.
The last test prints the geometry x precision table, asserts that the reported plans covered the plan space and that every negative
control (a reference with the last channel block or the last tap dropped, moved by one pixel tile, or without the bias) failed."""
import collections
import math

import pytest
import torch

from oracle import conv_ref as R
from test_gpu_conv_sweep import GUARD, TOL, TOL_STATS, _cw, _snapshot, _stats_err, _t, _untouched_outside

pytestmark = pytest.mark.gpu

# N, H, W, Cin, Cout, k (3x3 pad 1 or 1x1 pad 0).  Plans at 132 SMs (H100 SXM) -- the test asserts coverage from the plans the
# library reports, not these:
#   tc2 nt64 TN8 (4x4, padding CTA, 17 % 8), TN8 2x2, TN128 1x1 split 2, TN32 2x2 split 8, TN4 8x4 split 4, TN2 4x16,
#   tc2 TN1 2x32 (padding CTA), 8x16 with 3-stage A rings (split 4 / padding CTA / 9 tiles), 16x16, tc2 nt128 (34 / 48 tiles),
#   tc1 4x32 1x1 (padding CTA), tc1 4x32 128 channels, tc1 2x64 (its 3x3 halo exceeds 208 rows), tc1 1x128, tc1 nt128 (85 tiles),
#   tc1 1x128 over 256 columns.
GEOMS = [
    (17, 4, 4, 64, 64, 1), (9, 2, 2, 64, 128, 3), (1, 1, 1, 128, 64, 1), (1, 2, 2, 512, 64, 1), (1, 8, 4, 256, 64, 1),
    (1, 4, 16, 64, 64, 1), (3, 2, 32, 64, 64, 3), (1, 8, 16, 192, 128, 3), (5, 8, 16, 512, 192, 3), (3, 24, 16, 192, 128, 3),
    (2, 16, 16, 64, 64, 3), (17, 16, 16, 64, 256, 1), (2, 32, 96, 256, 256, 3), (1, 12, 32, 64, 64, 1), (2, 12, 32, 128, 128, 3),
    (1, 2, 64, 64, 64, 3), (1, 1, 128, 64, 64, 3), (17, 5, 128, 64, 128, 3), (2, 3, 256, 192, 128, 3),
]
REFUSED = [(1, 6, 16, 64, 64, 3), (2, 8, 12, 64, 64, 3)]      # neither tiling runs them
CAPS = (1, 5, 7)
PRECS = ("f16x3", "bf16x3")

RECORDS = []                                   # dict(geom, prec, call, plan, ratio)
CAP_ITEMS = {}                                 # geometry -> {cap: (clusters, work items)}
CONTROLS = collections.defaultdict(list)       # control -> [failed as it must]
DONE = set()


def _dev():
    return torch.device("cuda:0")


def _prec(name):
    from marconet_b200 import ops
    return {"f16x3": ops.PREC_F16X3_TC, "bf16x3": ops.PREC_BF16X3_TC}[name]


@pytest.fixture
def restore_cap():
    """Restores the CTA cap: ops.graph_key() includes it, so a leaked cap would also change later tests' captured graphs."""
    from marconet_b200 import ops
    old = ops.MAX_CTAS
    try:
        yield ops.set_max_ctas
    finally:
        ops.set_max_ctas(old)


def _guarded(n, oh, ow, c):
    """An NHWC channel slice [n, oh, ow, c] of a wider buffer with a guard sample after it: NaN in its own elements (every one must
    be written), GUARD everywhere else (must stay)."""
    big = torch.full((n + 1, oh, ow, c + 64), GUARD, device=_dev())
    y = big[:n, :, :, 32:32 + c]
    y.fill_(float("nan"))
    return y


def _input(n, h, w, cin, seed):
    """x: a channel slice of a wider buffer whose other channels hold NaN (a read outside [0, Cin) poisons the output)."""
    buf = torch.full((n, h, w, cin + 64), float("nan"), device=_dev())
    x = buf[..., 32:32 + cin]
    x.copy_(_t(n, h, w, cin, seed=seed, scale=1.5, shift=0.1))
    return x


def _epilogue(gi, n, oh, ow, cout):
    """The full epilogue: bias, per-sample out_scale (a column view of a wider buffer), residual (broadcast over the batch on odd
    geometries), LReLU with gain, y2_scale, ragged valid_w including 1."""
    vw = [[max(1, ow - 1), 1, ow, ow // 2 + 1][i % 4] for i in range(n)]
    bcast = gi % 2 == 1
    return dict(bias=_t(cout, seed=100 + gi), out_scale=_t(n, 2 * cout, seed=200 + gi, scale=0.3, shift=1.0)[:, cout:],
                residual=_t(1 if bcast else n, oh, ow, cout, seed=300 + gi), res_broadcast=bcast, act=R.ACT_LRELU02, gain=2 ** 0.5,
                y2_scale=_t(n, cout, seed=400 + gi), valid_w=torch.tensor(vw, dtype=torch.int32, device=_dev()))


def _ref(x0, cw, k, epi=None, gn=None, w=None):
    epi = dict(epi or {})
    act, gain = epi.pop("act", 0), epi.pop("gain", 1.0)
    return R.conv_ref_full(x0, cw.w if w is None else w, k, k, (1, 1), (k // 2, k // 2), gn=gn, act=act, gain=gain, **epi)


def _conv(x, cw, k, prec, y, epi=None, y2=None, **kw):
    """ops.conv2d into the guarded y (and y2): refills them with NaN first; returns (plan, statistics or None)."""
    from marconet_b200 import ops
    plan = {}
    y.fill_(float("nan"))
    if y2 is not None:
        y2.fill_(float("nan"))
    opts = dict(epi or {})
    if y2 is None:
        opts.pop("y2_scale", None)
    res = ops.conv2d(x, cw, k, k, pad=(k // 2, k // 2), out=y, out2=y2, precision=prec, plan=plan, **opts, **kw)
    torch.cuda.synchronize()
    return plan, (res[1] if kw.get("gn_stats") else None)


def _moved(t, plan):
    """t [N, OH, OW, ...] moved by one pixel tile: TW columns, else TH rows, else TN samples."""
    n, oh, ow = t.shape[:3]
    if ow > plan["TW"]:
        return t.roll(plan["TW"], 2)
    if oh > plan["TH"]:
        return t.roll(plan["TH"], 1)
    return t.roll(plan["TN"], 0)


def _controls(got, ref, x0, cw, k, cin, epi, plan, tol):
    """References that must fail the comparison; one is skipped where it equals the true reference (a single pixel tile)."""
    taps = k * k
    w_cb = cw.w.clone().view(taps, cin, -1)
    w_cb[:, cin - 64:] = 0
    w_tap = cw.w.clone().view(taps, cin, -1)
    w_tap[taps - 1] = 0
    bad = dict(last_channel_block=_ref(x0, cw, k, epi, w=w_cb.view(taps * cin, -1)),
               last_tap=_ref(x0, cw, k, epi, w=w_tap.view(taps * cin, -1)),
               moved_tile={key: _moved(ref[key], plan) for key in ("y", "bound")},
               no_bias=_ref(x0, cw, k, {key: v for key, v in epi.items() if key != "bias"}))
    for name, b in bad.items():
        if torch.equal(b["y"], ref["y"]):
            continue
        CONTROLS[name].append(R.ratio(got, b["y"], b["bound"], tol) > 1.0)


def _check(got, ref, key, tol, where):
    r = R.ratio(got, ref[key], ref["bound" if key == "y" else "bound2"], tol)
    assert r <= 1.0, f"{where} {key}: error / tolerance {r:.3g}"
    return r


def _plan_str(p):
    return (f"{p['kernel']} nt{p['nt']} {p['TN']}x{p['TH']}x{p['TW']} ks{p['splits']} cs{p['cs']} mt{p['m_tiles']} "
            f"hs{p['hstages']}/bs{p['bstages']} items{p['work_items']}")


def _run_geometry(gi, prec_name, set_cap):
    from marconet_b200 import ops
    n, h, w, cin, cout, k = GEOMS[gi]
    prec, tol = _prec(prec_name), TOL[_prec(prec_name)]
    oh, ow = h, w
    where = f"{GEOMS[gi]} {prec_name}"
    x = _input(n, h, w, cin, seed=gi)
    x0 = x.clone()
    cw = _cw(cout, cin, k, 10 + gi, f"plan_space.{gi}")
    y, y2 = _guarded(n, oh, ow, cout), _guarded(n, oh, ow, cout)
    snaps = [_snapshot(y), _snapshot(y2)]
    epi = _epilogue(gi, n, oh, ow, cout)
    ops.poll_range(_dev(), reroute=False)           # forget flags raised before this geometry

    def record(call, plan, ratio):
        RECORDS.append(dict(geom=gi, prec=prec_name, call=call, plan=plan, ratio=ratio, k=k, n=n))

    # plain
    plan, _ = _conv(x, cw, k, prec, y)
    assert plan["kernel"] in ("tc1", "tc2"), plan
    ref0 = _ref(x0, cw, k)
    record("plain", plan, _check(y, ref0, "y", tol, where + " plain"))
    assert _untouched_outside(snaps[0]), f"{where} plain: bytes outside the output slice changed"
    plain = [y.clone()]
    # full epilogue
    plan_e, _ = _conv(x, cw, k, prec, y, epi, y2=y2)
    ref = _ref(x0, cw, k, epi)
    record("epilogue", plan_e, max(_check(y, ref, "y", tol, where + " epilogue"), _check(y2, ref, "y2", tol, where + " epilogue")))
    assert all(_untouched_outside(s) for s in snaps), f"{where} epilogue: bytes outside the output slices changed"
    full = [y.clone(), y2.clone()]
    if prec_name == "f16x3":
        _controls(y, ref, x0, cw, k, cin, epi, plan_e, tol)
    # fused GroupNorm input + epilogue statistics: halo tiling, one sample per tile
    gn_out = None
    one_sample_halo = plan["kernel"] == "tc2" and plan["TN"] == 1
    if one_sample_halo:
        # mean / rstd as the call receives them (mn_groupnorm_stats itself takes no 192-channel maps)
        mr = R.groupnorm_stats64(x0, valid_w=epi["valid_w"].tolist()).float()
        gn = (mr, _t(cin, seed=500 + gi, scale=0.3, shift=1.0), _t(cin, seed=600 + gi, scale=0.2))
        gn0 = tuple(t.clone() for t in gn)
        plan_g, st = _conv(x, cw, k, prec, y, epi, y2=y2, gn=gn, gn_stats=True)
        assert plan_g["gn_fused"] and plan_g["gn_stats_out"], plan_g
        ref_g = _ref(x0, cw, k, epi, gn=gn0)
        r = max(_check(y, ref_g, "y", tol, where + " gn"), _check(y2, ref_g, "y2", tol, where + " gn"))
        e = _stats_err(st, R.groupnorm_stats64(y, valid_w=epi["valid_w"].tolist()))
        assert e <= TOL_STATS, f"{where} gn: epilogue GroupNorm statistics off by {e:.3g}"
        assert all(_untouched_outside(s) for s in snaps), f"{where} gn: bytes outside the output slices changed"
        record("gn", plan_g, r)
        gn_out = (gn, [y.clone(), y2.clone()], st.clone())
        # the second output through per-sample pointers into guarded buffers (shuffled order)
        blk, guard = oh * ow * cout, 1024
        big = torch.full((n * (blk + guard) + guard,), GUARD, device=_dev())
        dst = [big[guard + i * (blk + guard):guard + i * (blk + guard) + blk] for i in range(n)]
        order = list(range(n))[::-1]
        for b in dst:
            b.fill_(float("nan"))
        ptrs = torch.tensor([dst[order[i]].data_ptr() for i in range(n)], dtype=torch.int64, device=_dev())
        plan_p = {}
        y.fill_(float("nan"))
        ops.conv2d(x, cw, k, k, pad=(k // 2, k // 2), out=y, out2_ptrs=ptrs, precision=prec, plan=plan_p, **epi)
        torch.cuda.synchronize()
        got2 = torch.stack([dst[order[i]].view(oh, ow, cout) for i in range(n)])
        r = max(_check(y, ref, "y", tol, where + " y2_ptrs"), _check(got2, ref, "y2", tol, where + " y2_ptrs"))
        guards = [big[:guard]] + [big[guard + i * (blk + guard) + blk:guard + (i + 1) * (blk + guard)] for i in range(n)]
        assert all(bool((g == GUARD).all()) for g in guards), f"{where}: a store landed outside its y2_ptrs destination"
        record("y2_ptrs", plan_p, r)
    assert ops.poll_range(_dev(), reroute=False) == []
    if prec_name != "f16x3":
        return
    # CTA caps: the same bits from fewer clusters walking more work items
    items = CAP_ITEMS.setdefault(gi, {})
    try:
        for c in CAPS:
            set_cap(c)
            pc, _ = _conv(x, cw, k, prec, y)
            assert torch.equal(y, plain[0]), f"{where} plain at cap {c}: output differs from the uncapped call"
            pc, _ = _conv(x, cw, k, prec, y, epi, y2=y2)
            assert torch.equal(y, full[0]) and torch.equal(y2, full[1]), f"{where} epilogue at cap {c}: output differs from the uncapped call"
            assert pc["ctas"] == pc["cs"] * min(max(1, c // pc["cs"]), pc["work_items"]), pc
            items[c] = (pc["ctas"] // pc["cs"], pc["work_items"])
            if gn_out is not None:
                gn, (gy, gy2), gst = gn_out
                _, st = _conv(x, cw, k, prec, y, epi, y2=y2, gn=gn, gn_stats=True)
                assert torch.equal(y, gy) and torch.equal(y2, gy2), f"{where} gn at cap {c}: output differs from the uncapped call"
                # fp64 atomics in another order: the sums agree to ~1e-16 relative, the fp32 mean / rstd made of them to one rounding
                assert torch.allclose(st, gst, rtol=2.0 ** -23, atol=0), f"{where} gn at cap {c}: statistics differ"
            assert all(_untouched_outside(s) for s in snaps), f"{where} at cap {c}: bytes outside the output slices changed"
    finally:
        set_cap(0)
    assert items[1][0] == 1, items
    print(f"\n{where}: at cap 1 one cluster ran all {items[1][1]} work items ({_plan_str(plan_e)})")


@pytest.mark.parametrize("prec_name", PRECS)
@pytest.mark.parametrize("gi", range(len(GEOMS)), ids=["x".join(map(str, g[:3])) + f"_{g[3]}-{g[4]}_k{g[5]}" for g in GEOMS])
def test_geometry_matches_fp64(restore_cap, gi, prec_name):
    _run_geometry(gi, prec_name, restore_cap)
    DONE.add((gi, prec_name))


@pytest.mark.parametrize("gi", [i for i, g in enumerate(GEOMS) if g[:3] in ((1, 1, 1), (1, 2, 2), (1, 8, 4), (5, 8, 16))])
def test_split_k_under_a_small_workspace(gi):
    """The planned split needs ks * M * Cout floats of workspace: with room for half of them the plan halves the split, with room
    for one slice it does not split at all.  The full epilogue runs in the split-K reduce."""
    from marconet_b200 import ops
    n, h, w, cin, cout, k = GEOMS[gi]
    x = _input(n, h, w, cin, seed=50 + gi)
    x0 = x.clone()
    cw = _cw(cout, cin, k, 60 + gi, f"plan_space.ws{gi}")
    y, y2 = _guarded(n, h, w, cout), _guarded(n, h, w, cout)
    epi = _epilogue(gi, n, h, w, cout)
    ref = _ref(x0, cw, k, epi)
    plan, _ = _conv(x, cw, k, ops.PREC_F16X3_TC, y, epi, y2=y2)
    ks = plan["splits"]
    assert ks > 1, plan
    slice_bytes = n * h * w * cout * 4
    for want in dict.fromkeys((ks // 2, 1)):
        room = want
        with ops.use_workspace(torch.empty(room * slice_bytes // 4, device=_dev())):
            p, _ = _conv(x, cw, k, ops.PREC_F16X3_TC, y, epi, y2=y2)
        assert p["splits"] == want, (ks, p)
        where = f"{GEOMS[gi]} workspace for {room} slice(s)"
        RECORDS.append(dict(geom=gi, prec="f16x3", call=f"ws{room}", plan=p, k=k, n=n,
                            ratio=max(_check(y, ref, "y", TOL[1], where), _check(y2, ref, "y2", TOL[1], where))))


def _refused_cases():
    return [("geometry", g) for g in REFUSED] + [("x channel offset 1", (2, 16, 16, 64, 64, 3))]


@pytest.mark.parametrize("what,geom", _refused_cases(), ids=["6x16", "8x12", "misaligned_x"])
def test_refused_geometries(monkeypatch, what, geom):
    """An explicit tensor-core precision raises with the plan's reason for both tilings; the default precision runs the fp32
    kernel, which matches fp64."""
    from marconet_b200 import ops
    monkeypatch.setattr(ops, "TC_MIN_FLOP", 0.0)           # the fall-back must come from the plan, not from the launch size
    n, h, w, cin, cout, k = geom
    buf = torch.full((n, h, w, cin + 64), float("nan"), device=_dev())
    off = 1 if what.startswith("x channel") else 32
    x = buf[..., off:off + cin]
    x.copy_(_t(n, h, w, cin, seed=70))
    x0 = x.clone()
    cw = _cw(cout, cin, k, 71, f"plan_space.refused_{h}x{w}_{off}")
    y = _guarded(n, h, w, cout)
    with pytest.raises(RuntimeError, match=r"halo tiling: .*; per-tap tiling: "):
        ops.conv2d(x, cw, k, k, pad=(k // 2, k // 2), out=y, precision=ops.PREC_F16X3_TC)
    plan = {}
    assert ops.default_precision() != ops.PREC_FP32_SIMT
    ops.conv2d(x, cw, k, k, pad=(k // 2, k // 2), out=y, plan=plan)
    torch.cuda.synchronize()
    assert plan["kernel"] in ("simt", "small"), plan
    _check(y, _ref(x0, cw, k), "y", TOL[0], f"{geom} {what}: fp32 fall-back")


def test_pdl_off_chain_at_cap_1(restore_cap):
    """groupnorm_stats -> conv with the fused GroupNorm and epilogue statistics -> split-K conv reading it -> conv with tiles of
    several samples reading that -> per-tap conv reading that, on one stream without synchronisation, at cap 1 (the dependents'
    CTAs wait beside the running kernel): PDL on, PDL off and a synchronisation after every call give the same bits."""
    from marconet_b200 import _lib, ops
    lib = _lib.load()
    prec = ops.PREC_F16X3_TC
    x = _t(5, 8, 16, 64, seed=80, scale=1.5, shift=0.2)
    cws = [_cw(512, 64, 3, 81, "plan_space.chain1"), _cw(192, 512, 3, 82, "plan_space.chain2"),
           _cw(64, 192, 1, 83, "plan_space.chain3"), _cw(64, 64, 3, 84, "plan_space.chain4")]
    gamma, beta = _t(64, seed=85, scale=0.3, shift=1.0), _t(64, seed=86, scale=0.2)
    bias = [_t(c.cout, seed=87 + i) for i, c in enumerate(cws)]
    plans = [{} for _ in cws]

    def chain(sync):
        step = (lambda: torch.cuda.synchronize()) if sync else (lambda: None)
        mr = ops.groupnorm_stats(x)
        step()
        y1, st = ops.conv2d(x, cws[0], 3, 3, pad=(1, 1), bias=bias[0], gn=(mr, gamma, beta), gn_stats=True, precision=prec, plan=plans[0])
        step()
        y2 = ops.conv2d(y1, cws[1], 3, 3, pad=(1, 1), bias=bias[1], act=ops.ACT_LRELU02, precision=prec, plan=plans[1])
        step()
        y3 = ops.conv2d(y2.view(40, 4, 4, 192), cws[2], 1, 1, bias=bias[2], precision=prec, plan=plans[2])
        step()
        y4 = ops.conv2d(y3.view(5, 1, 128, 64), cws[3], 3, 3, pad=(1, 1), bias=bias[3], precision=prec, plan=plans[3])
        torch.cuda.synchronize()
        return [mr, y1, y2, y3, y4], st

    restore_cap(1)
    old = lib.mn_set_pdl(1)
    try:
        on, st_on = chain(False)
        lib.mn_set_pdl(0)
        off, st_off = chain(False)
        lib.mn_set_pdl(1)
        synced, st_sync = chain(True)
    finally:
        lib.mn_set_pdl(old)
    assert plans[0]["gn_fused"] and plans[0]["gn_stats_out"], plans[0]
    assert plans[1]["kernel"] == "tc2" and plans[1]["splits"] > 1, plans[1]
    assert plans[2]["kernel"] == "tc2" and plans[2]["TN"] > 1, plans[2]
    assert plans[3]["kernel"] == "tc1", plans[3]
    assert all(p["ctas"] == p["cs"] for p in plans), plans
    # statistics (step 1 and the epilogue's) are fp64 atomics in some order: equal to one fp32 rounding of the mean / rstd
    for i, (a, b, c) in enumerate(zip([st_on] + on, [st_off] + off, [st_sync] + synced)):
        if i < 2:
            assert torch.allclose(a, b, rtol=2.0 ** -23, atol=0) and torch.allclose(a, c, rtol=2.0 ** -23, atol=0), \
                f"{'epilogue' if i == 0 else 'step 1'} statistics differ beyond one fp32 rounding"
        else:
            assert torch.equal(a, b) and torch.equal(a, c), f"chain step {i}: PDL on / off / synchronised outputs differ"
    # and the chain itself is right: its last output against fp64 of the previous step's output
    ref = R.conv_ref_full(synced[3].view(5, 1, 128, 64), cws[3].w, 3, 3, (1, 1), (1, 1), bias=bias[3])
    _check(synced[4], ref, "y", TOL[1], "chain step 5")


def test_coverage_and_negative_controls(restore_cap):
    """Runs any geometry this session skipped, prints the table, asserts plan-space coverage and that every control failed."""
    for gi in range(len(GEOMS)):
        for p in PRECS:
            if (gi, p) not in DONE:
                _run_geometry(gi, p, restore_cap)
                DONE.add((gi, p))
    print("\ngeometry x precision: reported plan (first call) / calls / worst error-to-tolerance ratio / clusters:items at caps "
          + ",".join(map(str, CAPS)))
    by = collections.defaultdict(list)
    for r in RECORDS:
        by[(r["geom"], r["prec"])].append(r)
    for (gi, p), rs in sorted(by.items()):
        caps = " ".join(f"{c}:{a}/{b}" for c, (a, b) in sorted(CAP_ITEMS.get(gi, {}).items())) if p == "f16x3" else ""
        calls = ",".join(r["call"] for r in rs)
        print(f"{str(GEOMS[gi]):28s} {p:7s} {_plan_str(rs[0]['plan']):52s} {calls:28s} {max(r['ratio'] for r in rs):7.3f}  {caps}")
    print("negative controls (failed as they must):", {k: f"{sum(v)}/{len(v)}" for k, v in sorted(CONTROLS.items())})
    plans = [(r["plan"], r["k"], r["n"]) for r in RECORDS]
    seen = collections.defaultdict(set)
    for p, k, n in plans:
        seen["kernel"].add(p["kernel"])
        seen["nt"].add(p["nt"])
        seen["TN>1"].add(p["TN"] > 1)
        seen["ksplit"].add(p["splits"])
        seen["cs"].add(p["cs"])
        seen["padding CTA"].add(p["cs"] == 2 and p["m_tiles"] % 2 == 1)
        seen["N % TN != 0"].add(n % p["TN"] != 0)
        seen["hstages"].add(p["hstages"])
        seen["bstages"].add(p["bstages"])
        seen["TH*TW"].add(p["TH"] * p["TW"])
        seen["kernel x k"].add((p["kernel"], k))
    need = {"kernel": {"tc1", "tc2"}, "nt": {64, 128}, "TN>1": {True, False}, "ksplit": {1, 2, 4, 8}, "cs": {1, 2},
            "padding CTA": {True}, "N % TN != 0": {True}, "hstages": {2, 3}, "bstages": {3, 4}, "TH*TW": {1, 4, 16, 32, 64, 128},
            "kernel x k": {("tc1", 1), ("tc1", 3), ("tc2", 1), ("tc2", 3)}}
    for key, want in need.items():
        assert want <= seen[key], f"{key}: the reported plans cover {sorted(seen[key], key=str)}, not {sorted(want, key=str)}"
    assert any(items[1][1] > 1 for items in CAP_ITEMS.values()), CAP_ITEMS
    for name in ("last_channel_block", "last_tap", "moved_tile", "no_bias"):
        assert CONTROLS[name], f"control {name}: no geometry suited it"
        assert all(CONTROLS[name]), f"control {name} passed the comparison on {CONTROLS[name].count(False)} geometries"
