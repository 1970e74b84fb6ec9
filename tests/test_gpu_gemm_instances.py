"""gemm_bf16x3_kernel one instantiation and store path at a time: every case of tests/gemm_ref.py's table against the
fp64 emulation of the kernel's split passes at the case's emu_gate() and against true fp64 at GATE, run twice for identical bits,
with sentinel rows / columns around the output that must stay untouched.  Every conv case first asserts its plan with
ops.conv_plan; the plans and tile counts assume the 132 SMs of an H100 SXM.  tests/test_cpu_gemm_reference.py checks
that each case's inputs tell the planted mistakes apart."""
import ctypes
import math

import pytest
import torch

import gemm_ref as ref
from occformer_b200 import ops
from util import assert_close, parity_log, rejected, same_bits, sentinel, untouched

pytestmark = pytest.mark.gpu


def _check(out, true, emu, what, emu_gate):
    """out against the emulation at emu_gate and (true given) true fp64 at GATE; logs the least tolerance that would
    pass both criteria of assert_close against the emulation (the figure emu_gate() is set from)"""
    a, b = out.detach().double(), emu.detach().double().reshape(out.shape)
    d = (a - b).abs()
    need = max(float(d.max() / b.abs().max()), float((d / (b.pow(2).mean().sqrt() + b.abs())).max()))
    parity_log(f"[emulation] {what}: least passing tol {need:.3e}")
    assert_close(a, b, emu_gate, f"{what} vs emulation")
    if true is not None:
        assert_close(a, true.reshape(out.shape), ref.GATE, f"{what} vs fp64")


# ------------------------------------------------------------------------------------------------ plain GEMM
def _gemm(c, a_s, w_s, bias, res, dev, split_out=False):
    """one occ_gemm_bf16x3 launch into rows [0, M) of an (M + 3, N) sentinel buffer (from 4 bytes in when the case's
    output is misaligned) -> (output view, the rest of the buffer)"""
    M, N, K = c["M"], c["N"], c["K"]
    buf = sentinel(M + 3, N, dev)
    flat = buf.view(-1)
    out = flat[1:1 + M * N].view(M, N) if c["mis_out"] else buf[:M]
    if bias is not None and c["mis_bias"]:
        bb = torch.empty(N + 1, device=dev)
        bb[1:] = bias
        bias = bb[1:]
        assert bias.data_ptr() % 16 == 4
    ops._call("occ_gemm_bf16x3", a_s, w_s, out, M, N, K, bias, res, c["act"], int(split_out))
    return out, (torch.cat([flat[:1], flat[1 + M * N:]]) if c["mis_out"] else buf[M:])


def _gemm_operands(c, dev):
    a, w, bias, res = ref.gemm_inputs(c)
    cu = lambda t: None if t is None else t.to(dev)  # noqa: E731
    return cu(a), cu(w), cu(bias), cu(res)


@pytest.mark.parametrize("name", ref.GEMM_CASES)
def test_gemm(cuda, name):
    c = ref.GEMM_CASES[name]
    a, w, bias, res = _gemm_operands(c, cuda)
    a_s, w_s = ops.to_split(a), ops.split_weight(w)
    true, emu = ref.gemm_ref(a, w, bias, res, c["act"])
    out, rest = _gemm(c, a_s, w_s, bias, res, cuda)
    torch.cuda.synchronize()
    untouched(rest, f"gemm {name}")
    _check(out, true, emu, f"gemm {name} [{ref.gemm_label(c)}]", ref.emu_gate(c["K"] // 32))
    again, _ = _gemm(c, a_s, w_s, bias, res, cuda)
    same_bits(again, out, f"gemm {name}")
    if c["split_out"]:
        out_s, rest = _gemm(c, a_s, w_s, bias, res, cuda, split_out=True)
        untouched(rest, f"gemm {name} split_out")
        same_bits(out_s, ops.to_split(out.contiguous()), f"gemm {name}: split_out != to_split(fp32 output)")


@pytest.mark.parametrize("name", ref.GEMM_CASES)
def test_gemm_single_pass(cuda, name):
    c = ref.GEMM_CASES[name]
    a, w, bias, res = _gemm_operands(c, cuda)
    a_s, w_s = ops.to_split(a), ops.split_weight(w)
    _, emu = ref.gemm_ref(a, w, bias, res, c["act"], passes=1)
    with ops.precision("bf16"):
        out, rest = _gemm(c, a_s, w_s, bias, res, cuda)
        again, _ = _gemm(c, a_s, w_s, bias, res, cuda)
    untouched(rest, f"bf16 gemm {name}")
    _check(out, None, emu, f"bf16 gemm {name}", ref.emu_gate(c["K"] // 32, passes=1))
    same_bits(again, out, f"bf16 gemm {name}")


# ------------------------------------------------------------------------------------------------ conv
_REF = {}


def _conv_ref(base, dev, passes=3):
    """(x, w, true, emulated) of a conv base on dev, fp64 raw outputs, computed once per base"""
    key = (base, passes)
    if key not in _REF:
        _REF.clear()  # the MT2 base's references take ~0.5 GB: keep one base at a time
        x, w = ref.conv_inputs(base)
        B, X, Y, Z, Cin, Cout, k, stride, dil = ref.CONV_BASES[base]
        x, w = x.to(dev), w.to(dev)
        _REF[key] = (x, w) + ref.conv_contract(x, w, stride, dil, passes)
    return _REF[key]


def _workspace(dev):
    return torch.zeros(ops.lib().occ_conv_workspace_bytes(), dtype=torch.uint8, device=dev)


def _conv(c, x_s, w2, bias, res, stats, ws, dev, split_out=None):
    """one occ_conv_bf16x3 / occ_conv_slice_bf16x3 launch of case c -> (output (rows, Cout) view, untouched part)"""
    B, X, Y, Z, Cin, _, k, stride, dil = ref.CONV_BASES[c["base"]]
    N = c["cols"]
    rows = B * math.prod(ref.conv_out_shape(c["base"]))
    so = int(c["split_out"] if split_out is None else split_out)
    wsa = (ws, ws.numel()) if ws is not None else (None, 0)
    common = (B, X, Y, Z, Cin, N, *k, stride, dil, bias, res, c["act"], so, stats, c["cpg"], *wsa)
    if c["out"] == "slice":
        buf = sentinel(rows, c["ldo"], dev)
        ops._call("occ_conv_slice_bf16x3", x_s, w2, buf, c["ldo"], c["off"], *common)
        lo, hi = c["off"], c["off"] + N
        return buf[:, lo:hi], torch.cat([buf[:, :lo].reshape(-1), buf[:, hi:].reshape(-1)])
    buf = sentinel(rows + 3, N, dev)
    flat = buf.view(-1)
    if c["out"] == "misaligned":
        out = flat[1:1 + rows * N].view(rows, N)
        ops._call("occ_conv_bf16x3", x_s, w2, out, *common)
        return out, torch.cat([flat[:1], flat[1 + rows * N:]])
    out = buf[:rows]
    ops._call("occ_conv_bf16x3", x_s, w2, out, *common)
    return out, buf[rows:]


def _conv_setup(c, dev, passes=3):
    x, w, true, emu = _conv_ref(c["base"], dev, passes)
    N = c["cols"]
    B = x.shape[0]
    rows = true[..., 0].numel()
    bias, res = ref.epilogue_inputs(rows, N, c)
    bias = None if bias is None else bias.to(dev)
    res = None if res is None else res.to(dev)
    x_s = ops.to_split(x)
    w2 = ops.repack_conv_weight(w[:N])[0]
    raw_t, raw_e = true[..., :N].reshape(rows, N), emu[..., :N].reshape(rows, N)
    return B, rows, x_s, w2, bias, res, raw_t, raw_e


def _assert_plan(c):
    B, X, Y, Z, Cin, _, k, stride, dil = ref.CONV_BASES[c["base"]]
    plan, _, splitk_ok = ref.conv_case_plan(c)
    want = (ref.BM * plan["mt"], plan["bn"], plan["stages"], plan["splits"])
    assert ops.conv_plan(B, X, Y, Z, Cin, c["cols"], k, stride, dil, splitk_ok) == want, f"{c}: not the plan {want}"
    return plan


@pytest.mark.parametrize("name", ref.CONV_CASES)
def test_conv(cuda, name):
    c = ref.CONV_CASES[name]
    plan = _assert_plan(c)
    B, rows, x_s, w2, bias, res, raw_t, raw_e = _conv_setup(c, cuda)
    N, cpg = c["cols"], c["cpg"]
    ws = _workspace(cuda) if c["splitk"] else None
    stats = torch.zeros(B, N // cpg, 2, dtype=torch.float64, device=cuda) if cpg else None
    what = f"conv {name} [{ref.conv_label(c)}]"
    out, rest = _conv(c, x_s, w2, bias, res, stats, ws, cuda, split_out=False)
    torch.cuda.synchronize()
    untouched(rest, what)
    if ws is not None:
        assert int(ws.count_nonzero()) == 0, f"{what}: split-K counters left non-zero"
    ep = lambda y: ref.epilogue(y, bias, res, c["act"])  # noqa: E731
    nkb = ref.conv_nkb(c["base"])
    _check(out, ep(raw_t), ep(raw_e), what, ref.emu_gate(nkb))
    if cpg:
        st, se = ref.gn_stats(raw_t.view(B, -1, N), B, cpg), ref.gn_stats(raw_e.view(B, -1, N), B, cpg)
        _check(stats, None, se, f"{what} gn_stats", ref.stats_gate(nkb))
        assert_close(stats, st, 1e-4, f"{what} gn_stats vs fp64")
    again, _ = _conv(c, x_s, w2, bias, res, None, ws, cuda, split_out=False)
    same_bits(again, out, what)
    if ws is not None:
        assert int(ws.count_nonzero()) == 0, f"{what}: split-K counters left non-zero"
    if c["split_out"]:
        out_s, rest = _conv(c, x_s, w2, bias, res, None, ws, cuda)
        untouched(rest, f"{what} split_out")
        same_bits(out_s, ops.to_split(out.contiguous()), f"{what}: split_out != to_split(fp32 output)")
    assert plan["splits"] == 1 or ws is not None


@pytest.mark.parametrize("name", ["k331 cpg3", "splitK BN96"])
def test_conv_single_pass(cuda, name):
    c = ref.CONV_CASES[name]
    _assert_plan(c)
    B, rows, x_s, w2, bias, res, _, raw_e = _conv_setup(c, cuda, passes=1)
    ws = _workspace(cuda) if c["splitk"] else None
    with ops.precision("bf16"):
        out, rest = _conv(c, x_s, w2, bias, res, None, ws, cuda)
        again, _ = _conv(c, x_s, w2, bias, res, None, ws, cuda)
    untouched(rest, f"bf16 conv {name}")
    _check(out, None, ref.epilogue(raw_e, bias, res, c["act"]), f"bf16 conv {name}",
           ref.emu_gate(ref.conv_nkb(c["base"]), passes=1))
    same_bits(again, out, f"bf16 conv {name}")


def test_splitk_workspace_is_reset(cuda):
    """two different split-K convs back to back on one workspace leave it zero after each call; the first conv again on
    a fresh workspace gives the same bits"""
    ws = _workspace(cuda)
    outs = []
    for name in ("splitK BN32", "splitK BN128", "splitK BN32"):
        c = ref.CONV_CASES[name]
        assert _assert_plan(c)["splits"] > 1
        _, _, x_s, w2, bias, res, _, _ = _conv_setup(c, cuda)
        outs.append(_conv(c, x_s, w2, bias, res, None, ws, cuda)[0].clone())
        torch.cuda.synchronize()
        assert int(ws.count_nonzero()) == 0, f"{name}: split-K counters left non-zero"
    fresh = _conv(c, x_s, w2, bias, res, None, _workspace(cuda), cuda)[0]
    same_bits(outs[2], outs[0], "split-K conv after another conv on the same workspace")
    same_bits(fresh, outs[0], "split-K conv on a fresh workspace")


# ------------------------------------------------------------------------------------------------ tap tables
def _taps_arr(taps):
    flat = [int(v) for t in taps for v in t]
    return (ctypes.c_int * len(flat))(*flat)


@pytest.mark.parametrize("name", ref.TAP_CASES)
def test_conv_taps(cuda, name):
    B, X, Y, Z, Cin, Cout, taps, cpg = ref.TAP_CASES[name]
    x, w2 = (t.to(cuda) for t in ref.taps_inputs(name))
    true, emu, st, se = ref.conv_ref(x, w2, taps=taps, cpg=cpg)
    x_s, w_s = ops.to_split(x), ops.split_weight(w2)
    stats = torch.zeros(B, Cout // cpg, 2, dtype=torch.float64, device=cuda)
    what = f"conv_taps {name} [{ref.tap_label(name)}]"
    rows = B * X * Y * Z
    buf = sentinel(rows + 3, Cout, cuda)
    ops._call("occ_conv_taps_bf16x3", x_s, w_s, buf[:rows], B, X, Y, Z, Cin, Cout, len(taps), _taps_arr(taps), stats, cpg)
    torch.cuda.synchronize()
    untouched(buf[rows:], what)
    nkb = len(taps) * Cin // ref.BK
    _check(buf[:rows], true.view(rows, Cout), emu.view(rows, Cout), what, ref.emu_gate(nkb))
    _check(stats, None, se, f"{what} gn_stats", ref.stats_gate(nkb))
    same_bits(ops.conv_taps(x_s, w_s, taps).view(rows, Cout), buf[:rows], what)


def test_conv_taps_rejects_bad_tables(cuda):
    B, X, Y, Z, Cin, Cout = 1, 4, 4, 4, 32, 32
    x_s = torch.zeros(B, X, Y, Z, Cin, device=cuda)
    out = sentinel(B * X * Y * Z, Cout, cuda)
    for taps in ([(0, 0, 0)] * 29, [(0, 128, 0)], [(-128, 0, 0)], [(0, 0, 1), (0, 0, -200)]):
        w2 = torch.zeros(Cout, len(taps) * Cin, device=cuda)
        rejected("occ_conv_taps_bf16x3", x_s, w2, out, B, X, Y, Z, Cin, Cout, len(taps), _taps_arr(taps), None, 0,
                 buffers=(out,))
