"""tests/gemm_ref.py on the host: its true-fp64 part equals F.linear / F.conv3d / a hand-written tap sum, its emulation
stays within the dropped lo.lo' bound of the true result, the case table of tests/test_gpu_gemm_instances.py reaches
every instantiation and store path of gemm_bf16x3_kernel, and on each case's own inputs every applicable planted mistake
moves the emulated result by more than 10 x the case's emu_gate() (a k-block plant by more than 2 x).  A GPU failure then points at the kernel, and a case that cannot
tell a mistake apart fails here."""
import functools

import pytest
import torch
import torch.nn.functional as F

import gemm_ref as ref
from occformer_b200 import ops
from util import rel_err



def _bites(mutant, want, what, gate, times=10):
    r, need = rel_err(mutant, want), times * gate
    assert r > need, f"{what}: the planted mistake moves the result by only {r:.2e} (needs > {need:.1e})"


def _kb_times(m):
    return 2 if m in ref.KBLOCK_MISTAKES else 10


# ------------------------------------------------------------------------------------------------ the restatement
def test_split_is_split_weight():
    g = torch.Generator().manual_seed(ref.case_seed(1))
    x = torch.randn(64, 96, generator=g) * torch.logspace(-20, 20, 96)
    hi, lo = ref.split(x)
    packed = ops.split_weight(x).view(torch.bfloat16).view(64, 3, 64).double()
    assert torch.equal(hi, packed[:, :, :32].reshape(64, 96)) and torch.equal(lo, packed[:, :, 32:].reshape(64, 96))
    assert float(((hi + lo - x.double()).abs() / x.double().abs()).max()) <= 2.0 ** -17


def _act(y, act):
    return [lambda v: v, F.relu, lambda v: F.gelu(v, approximate="none"), F.silu][act](y)


@pytest.mark.parametrize("act", range(4))
def test_gemm_true_is_linear_and_emulation_within_lolo_bound(act):
    g = torch.Generator().manual_seed(ref.case_seed(2, act))
    a, w = torch.randn(70, 160, generator=g), torch.randn(50, 160, generator=g) * 160 ** -0.5
    bias, res = torch.randn(50, generator=g), torch.randn(70, 50, generator=g)
    true, emu = ref.gemm_ref(a, w, bias, res, act)
    want = _act(F.linear(a.double(), w.double(), bias.double()) + res.double(), act)
    assert rel_err(true, want) < 1e-14
    # true - emu = sum al.wl' + ea.w + (ah + al).ew, e = what hi + lo misses of an operand: bounded before the epilogue
    t0, e0 = ref.contract(a, w)
    (ah, al), (wh, wl) = ref.split(a), ref.split(w)
    ea, ew = a.double() - ah - al, w.double() - wh - wl
    bound = al.abs() @ wl.abs().t() + ea.abs() @ w.double().abs().t() + (ah + al).abs() @ ew.abs().t()
    assert bool(((t0 - e0).abs() <= bound * (1 + 1e-9) + 1e-14).all())
    assert float((t0 - e0).abs().max()) > 0  # the emulation is not the true product
    t1, e1 = ref.contract(a, w, passes=1)
    assert torch.equal(t1, t0) and rel_err(e1, ah @ wh.t()) == 0


@pytest.mark.parametrize("k,stride,dil", [((3, 3, 3), 1, 1), ((1, 3, 3), 2, 1), ((3, 1, 3), 1, 2), ((3, 3, 1), 2, 3)])
def test_conv_true_is_tap_sum(k, stride, dil):
    g = torch.Generator().manual_seed(ref.case_seed(3, *k, stride, dil))
    x, w = torch.randn(2, 7, 6, 5, 32, generator=g), torch.randn(40, 32, *k, generator=g)
    true, emu = ref.conv_contract(x, w, stride, dil)
    shape = tuple(ref.out_size(n, kk, stride, dil) for n, kk in zip((7, 6, 5), k))
    taps = ref.stencil_taps(k, dil)
    w2 = w.permute(0, 2, 3, 4, 1).reshape(40, len(taps), 32).double()
    assert rel_err(true, ref.tap_sum(x.double(), w2, taps, stride, shape)) < 1e-14
    (xh, xl), (wh, wl) = ref.split(x), ref.split(w2.float())
    want = ref.tap_sum(xh, wh, taps, stride, shape) + ref.tap_sum(xl, wh, taps, stride, shape) \
        + ref.tap_sum(xh, wl, taps, stride, shape)
    assert rel_err(emu, want) < 1e-14 and rel_err(emu, true) < 1e-4


def _naive_taps(x, w2, taps):
    """one output voxel at a time"""
    B, X, Y, Z, Cin = x.shape
    w = w2.double().view(w2.shape[0], len(taps), Cin)
    out = torch.zeros(B, X, Y, Z, w.shape[0], dtype=torch.float64)
    for b in range(B):
        for i in range(X):
            for j in range(Y):
                for l in range(Z):
                    for t, (dx, dy, dz) in enumerate(taps):
                        u, v, s = i + dx, j + dy, l + dz
                        if 0 <= u < X and 0 <= v < Y and 0 <= s < Z:
                            out[b, i, j, l] += w[:, t] @ x[b, u, v, s].double()
    return out


@pytest.mark.parametrize("name", ref.TAP_CASES)
def test_taps_true_is_naive_sum(name):
    B, X, Y, Z, Cin, Cout, taps, cpg = ref.TAP_CASES[name]
    x, w2 = ref.taps_inputs(name)
    true, emu, st, se = ref.conv_ref(x, w2, taps=taps, cpg=cpg)
    assert rel_err(true, _naive_taps(x, w2, taps)) < 1e-14 and rel_err(emu, true) < 1e-4
    assert rel_err(st, ref.gn_stats(true.view(B, -1, Cout), B, cpg)) == 0
    if any(abs(d) >= n for t in taps for d, n in zip(t, (X, Y, Z))):  # a tap entirely outside the grid adds nothing
        inside = [t for t in taps if all(abs(d) < n for d, n in zip(t, (X, Y, Z)))]
        keep = [i for i, t in enumerate(taps) if t in inside]
        w_in = w2.view(Cout, len(taps), Cin)[:, keep].reshape(Cout, -1)
        assert rel_err(ref.taps_contract(x, w_in, inside)[0], true) < 1e-14


def test_conv_plan_restatement_matches_the_documented_plans():
    """the plans tests/test_gpu_conv_tiles.py asserts on an H100 SXM, from the restated rules"""
    for (B, X, Y, Z, Cin, Cout, s), plan in [((4, 200, 200, 16, 128, 128, 1), (256, 128, 4, 1)),
                                             ((4, 200, 200, 16, 192, 192, 1), (256, 96, 4, 1)),
                                             ((4, 200, 200, 16, 128, 256, 2), (256, 128, 4, 1)),
                                             ((4, 100, 100, 8, 256, 256, 1), (256, 128, 4, 1)),
                                             ((4, 50, 50, 4, 512, 512, 1), (128, 128, 3, 1)),
                                             ((1, 101, 83, 16, 96, 128, 1), (256, 128, 4, 1))]:
        o = [(n - 1) // s + 1 for n in (X, Y, Z)]
        p = ref.conv_plan(B, *o, Cout, s, 27 * Cin // 32, True)
        assert (128 * p["mt"], p["bn"], p["stages"], p["splits"]) == plan


# ------------------------------------------------------------------------------------------------ the case table
def test_case_table_covers_every_instantiation_and_store_path():
    labels = ({ref.gemm_label(c) for c in ref.GEMM_CASES.values()} | {ref.conv_label(c) for c in ref.CONV_CASES.values()}
              | {ref.tap_label(n) for n in ref.TAP_CASES})
    assert ref.REQUIRED <= labels, f"not reached: {sorted(ref.REQUIRED - labels)}"
    assert len(ref.REQUIRED) == 19
    # every plain-GEMM instantiation and store path with more tiles than SMs (the persistent loop's later tiles), the
    # lean ones with more than two tiles per SM
    big = {}
    for c in ref.GEMM_BIG.values():
        big[ref.gemm_label(c)] = max(big.get(ref.gemm_label(c), 0), ref.gemm_tiles(c))
    assert set(big) == {x for x in ref.REQUIRED if "MT2" not in x and "split" not in x}
    assert all(t > ref.SMS for t in big.values())
    assert all(t > 2 * ref.SMS for lab, t in big.items() if lab.startswith("lean"))
    # a k-block count that is not a multiple of the ring depth, and one k-block per tile
    nkb = {ref.gemm_label(c): c["K"] // 32 for c in ref.GEMM_BIG.values()}
    assert nkb["lean BN128 TMA"] == 1 and nkb["lean BN64 TMA"] % ref.gemm_stages(64, 1)
    assert {c["M"] for c in ref.GEMM_EDGES.values()} == {1, 127, 128, 129, 257}
    # act 0-3 x bias x residual on every plain-GEMM instantiation and store path
    combos = {(ref.gemm_label(c), c["act"], c["bias"], c["residual"]) for c in ref.GEMM_EPI.values()}
    for lab in big:
        for act in range(4):
            assert {(b, r) for (l_, a, b, r) in combos if l_ == lab and a == act} >= {(True, False), (True, True)}
    assert {ref.gemm_bn(c["N"]) for c in ref.GEMM_SPLIT_OUT.values()} == {32, 64, 96, 128}


def test_conv_cases_reach_their_plans_and_edges():
    for name, c in ref.CONV_CASES.items():
        lab = ref.conv_label(c)
        assert ("MT2" in lab) == name.startswith("MT2") and ("split-K" in lab) == name.startswith("splitK"), name
    plan = ref.conv_case_plan(ref.CONV_CASES["k133 B3 cpg1"])[0]
    assert ref.CONV_BASES["k133 B3"][0] == 3 and plan["m_tiles"] * plan["n_tiles"] > ref.SMS
    ks = {ref.CONV_BASES[c["base"]][6] for c in ref.CONV_CASES.values()}
    assert {(1, 3, 3), (3, 1, 3), (3, 3, 1)} <= ks
    # the split-K boundaries: one inside a tap's Cin blocks, one at the start of a tap whose z index wraps to 0
    bounds = [b for n, c in ref.CONV_CASES.items() if n.startswith("splitK") for b in ref.split_boundaries(c)]
    assert any(cb != 0 for _, cb in bounds) and any(cb == 0 and t % 3 == 0 for t, cb in bounds)
    cpgs = {c["cpg"] for c in ref.CONV_CASES.values()} | {v[-1] for v in ref.TAP_CASES.values()}
    assert {1, 2, 3, 5, 6, 12, 16, 24, 48, 64, 96} <= cpgs
    assert ref.CONV_CASES["Cout192 cpg2"]["cols"] // 2 == ref.MAX_STAT_GROUPS
    gs = {c["cpg"] for n, c in ref.CONV_CASES.items() if n.startswith("splitK")}
    assert {5, 48} <= gs
    ntaps = {len(v[6]) for v in ref.TAP_CASES.values()}
    assert {1, 28} <= ntaps


# ------------------------------------------------------------------------------------------------ planted mistakes
@functools.lru_cache(maxsize=None)
def _conv_base(base):
    x, w = ref.conv_inputs(base)
    B, X, Y, Z, Cin, Cout, k, stride, dil = ref.CONV_BASES[base]
    return x, w, ref.conv_contract(x, w, stride, dil)[1]


@functools.lru_cache(maxsize=None)
def _conv_delta(base, mistake, splits):
    x, w, _ = _conv_base(base)
    B, X, Y, Z, Cin, Cout, k, stride, dil = ref.CONV_BASES[base]
    return ref.conv_mistake(x, w, stride, dil, 3, splits, mistake)


def _gemm_mistakes(c):
    out = list(ref.KBLOCK_MISTAKES) + ["last row dropped"]
    if c["N"] % 32:
        out.append("last partial column dropped")
    if c["act"] and c["bias"]:
        out.append("bias after the activation")
    if c["act"] and c["residual"]:
        out.append("residual after the activation")
    return out


@pytest.mark.parametrize("name", ref.GEMM_CASES)
def test_gemm_inputs_tell_planted_mistakes_apart(name):
    c = ref.GEMM_CASES[name]
    a, w, bias, res = ref.gemm_inputs(c)
    want = ref.gemm_ref(a, w, bias, res, c["act"])[1]
    gate = ref.emu_gate(c["K"] // 32)
    for m in _gemm_mistakes(c):
        _bites(ref.gemm_ref(a, w, bias, res, c["act"], mistake=m)[1], want, f"{name}: {m}", gate, _kb_times(m))


def _observable(c, mistake, splits):
    """whether a conv mistake can change the output at all: some tap it concerns reads inside the grid for some output
    voxel (in the grid of "tiny", X = Z = 1, every tap with a nonzero x or z offset reads only padding)"""
    B, X, Y, Z, Cin, _, k, stride, dil = ref.CONV_BASES[c["base"]]
    taps = ref.stencil_taps(k, dil)
    out = ref.conv_out_shape(c["base"])
    inside = lambda off: all(ref._range(o, n, stride, d) for o, n, d in zip(out, (X, Y, Z), off))  # noqa: E731
    if mistake in ref.KBLOCK_MISTAKES:
        return any(inside(taps[t]) for _, t, _ in ref._kblock_cols(len(taps) * Cin, splits, Cin // ref.BK))
    ax = "xyz".index(mistake.split()[3])
    idx = [(i, j, l) for i in range(k[0]) for j in range(k[1]) for l in range(k[2])]
    moved = lambda off: tuple(v + (a == ax) for a, v in enumerate(off))  # noqa: E731
    return any(inside(taps[t]) or inside(moved(taps[t])) for t, i in enumerate(idx) if i[ax] == k[ax] - 1)


def test_only_the_tiny_grid_hides_a_mistake():
    hidden = {(n, m) for n, c in ref.CONV_CASES.items() for m in ref.KBLOCK_MISTAKES + ref.TAP_MISTAKES
              if not _observable(c, m, ref.conv_case_plan(c)[0]["splits"])}
    assert hidden == {("tiny", m) for m in ref.KBLOCK_MISTAKES + ref.TAP_MISTAKES[::2]}


@pytest.mark.parametrize("name", ref.CONV_CASES)
def test_conv_inputs_tell_planted_mistakes_apart(name):
    c = ref.CONV_CASES[name]
    x, w, emu = _conv_base(c["base"])
    B, X, Y, Z, Cin, _, k, stride, dil = ref.CONV_BASES[c["base"]]
    N = c["cols"]
    plan = ref.conv_case_plan(c)[0]
    gate = ref.emu_gate(ref.conv_nkb(c["base"]))
    raw = emu[..., :N]
    rows = raw.numel() // N
    bias, res = ref.epilogue_inputs(rows, N, c)
    ep = lambda y, m=None: ref.epilogue(y.reshape(rows, N), bias, res, c["act"], m)  # noqa: E731
    want = ep(raw)
    for m in ref.KBLOCK_MISTAKES + ref.TAP_MISTAKES:
        if not _observable(c, m, plan["splits"]):
            continue
        d = _conv_delta(c["base"], m, plan["splits"])[..., :N]
        _bites(ep(raw + d), want, f"{name}: {m}", gate, _kb_times(m))
    em = ["last row dropped"] + (["last partial column dropped"] if N % 32 else []) \
        + (["bias after the activation"] if c["act"] and c["bias"] else []) \
        + (["residual after the activation"] if c["act"] and c["residual"] else [])
    for m in em:
        _bites(ep(raw, m), want, f"{name}: {m}", gate)
    if c["cpg"] and N // c["cpg"] >= 2:
        y = raw.reshape(B, -1, N)
        _bites(ref.gn_stats(y, B, c["cpg"], ref.STATS_MISTAKES[0]), ref.gn_stats(y, B, c["cpg"]), f"{name}: stats",
               ref.stats_gate(ref.conv_nkb(c["base"])))


@pytest.mark.parametrize("name", ref.TAP_CASES)
def test_taps_inputs_tell_planted_mistakes_apart(name):
    B, X, Y, Z, Cin, Cout, taps, cpg = ref.TAP_CASES[name]
    x, w2 = ref.taps_inputs(name)
    _, emu, _, se = ref.conv_ref(x, w2, taps=taps, cpg=cpg)
    _, bad, _, bad_s = ref.conv_ref(x, w2, taps=taps, cpg=cpg, mistake=ref.TAP_MISTAKES[0])
    nkb = len(taps) * Cin // ref.BK
    _bites(bad, emu, f"{name}: {ref.TAP_MISTAKES[0]}", ref.emu_gate(nkb))
    _bites(ref.conv_ref(x, w2, taps=taps, cpg=cpg, mistake=ref.STATS_MISTAKES[0])[3], se, f"{name}: stats",
           ref.stats_gate(nkb))
