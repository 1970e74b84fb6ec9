"""The pixel decoder's non-GEMM kernels one launch at a time against the fp64 reference of tests/neck_ref.py:
occ_ms_deform_attn, occ_neck_token_prep, occ_gn_upsample_add (the tiled x2 kernel and the general one) and occ_gn_stats.

Every case also checks what the whole-neck tests cannot see: the launch count of the entry point, bit-identical repeat
launches (all but occ_gn_stats, whose sums are fp64 atomics), S32 outputs that are bit for bit the split of the fp32
value, NaN sentinels in every output so that a row left unwritten fails, and rejected calls that raise, enqueue nothing
and leave every buffer as it was.  GroupNorm statistics fed to occ_gn_upsample_add are computed in fp64, so that kernel is
tested apart from occ_gn_stats.  tests/test_cpu_neck_reference.py checks the reference, and that these inputs tell planted
mistakes apart.

Gates (tests/util.assert_close, both criteria): GATE for fp32 results, GATE_S32 for decoded S32 outputs, also for the
token row offset by 1e3 x its spread and for the GroupNorm groups with mean / std = 100 on their own."""
import ctypes

import pytest
import torch

import neck_ref as ref
from oracle import port
from util import assert_close, launches, misaligned, rejected, same_bits, sentinel
from occformer_b200 import ops

pytestmark = pytest.mark.gpu

GATE, GATE_S32 = ref.GATE_F32, ref.GATE_S32


def _grids(grids):
    flat = [int(v) for g in grids for v in g]
    return (ctypes.c_int * len(flat))(*flat)


def _strides(strides):
    return (ctypes.c_float * len(strides))(*[float(s) for s in strides])


# ------------------------------------------------------------------------------------------------ occ_ms_deform_attn
def _msda(value, ow, grids, strides, B, E, H, head_ld, P=4):
    out = sentinel(value.shape[0], E, value.device)
    n = launches("occ_ms_deform_attn", value, value.shape[1], head_ld, ow, out, len(grids), B, _grids(grids),
                 _strides(strides), E, H, P)
    assert n == 1
    return out


def _port_fp32(value, ow, grids, strides, B, E, H, head_ld, P=4):
    """port.ms_deform_attn_core_3d (= multi_scale_deformable_attn_pytorch) in fp32 on the host, on level-major operands,
    with its reference points from port.grid_priors_3d as the port's decoder makes them"""
    L = len(grids)
    hd = E // H
    starts, ns = ref.level_starts(grids)
    sm = lambda t: torch.cat([t[B * s:B * (s + n)].reshape(B, n, *t.shape[1:]) for s, n in zip(starts, ns)], 1)  # noqa
    Nq = sum(ns)
    v = sm(value.cpu().view(-1, H, head_ld)[:, :, :hd].contiguous())
    o = sm(ow.cpu())
    off = o[..., :H * L * P * 3].reshape(B, Nq, H, L, P, 3)
    aw = o[..., H * L * P * 3:].reshape(B, Nq, H, L * P).softmax(-1).view(B, Nq, H, L, P)
    refs = torch.cat([port.grid_priors_3d(g, s) / (torch.tensor([[g[2], g[1], g[0]]], dtype=torch.float32) * s)
                      for g, s in zip(grids, strides)])
    norm = torch.tensor([[Z, Y, X] for (X, Y, Z) in grids], dtype=torch.float32)
    loc = refs[None, :, None, None, None, :] + off / norm[None, None, None, :, None, :]
    want = port.ms_deform_attn_core_3d(v, grids, loc, aw)
    return torch.cat([want[:, s:s + n].reshape(-1, E) for s, n in zip(starts, ns)])


@pytest.mark.parametrize("case", range(len(ref.MSDA_CASES)),
                         ids=lambda i: "L{}-E{}-H{}-B{}-rows{}".format(
                             len(ref.MSDA_CASES[i][0]), *ref.MSDA_CASES[i][2:5],
                             ref.MSDA_CASES[i][4] * sum(x * y * z for x, y, z in ref.MSDA_CASES[i][0])))
def test_ms_deform_attn_against_fp64(cuda, case):
    """every head_ld of the case gives the same bits; a padded layout has NaN in its pad columns, so a read of the pad
    poisons the output"""
    grids, strides, E, H, B, lds = ref.MSDA_CASES[case]
    hd = E // H
    ow = ref.ow_input(grids, B, H, seed=ref.case_seed(case, 2)).to(cuda)
    base = ref.value_input(grids, B, E, H, seed=ref.case_seed(case, 1)).to(cuda)
    want = ref.ms_deform_attn(base.double(), ow, grids, strides, B, E, H, coords="fp32")
    name = f"ms_deform_attn L{len(grids)} E{E} H{H} B{B} rows{base.shape[0]}"
    first = None
    for ld in lds:
        value = base
        if ld != hd:
            value = torch.full((base.shape[0], H, ld), float("nan"), device=cuda)
            value[:, :, :hd] = base.view(-1, H, hd)
            value = value.view(-1, H * ld)
        out = _msda(value, ow, grids, strides, B, E, H, ld)
        assert_close(ops.unsplit_weight(out), want, GATE_S32, f"{name} head_ld {ld} (S32)")
        same_bits(_msda(value, ow, grids, strides, B, E, H, ld), out, f"head_ld {ld}: repeat launch")
        if first is None:
            first = out
        else:
            same_bits(out, first, f"head_ld {ld} vs head_ld {lds[0]}")
    if base.shape[0] <= 20000:  # the port's own arithmetic, in fp32 on the host, with its zeros padding
        ow_c = ow.clone()
        n = H * len(grids) * 4 * 3
        ow_c[:, :n] = ow_c[:, :n].clamp(-1e4 - 50, 1e4 + 50)  # grid_sample's int conversion is not defined at 1e30
        got = ops.unsplit_weight(_msda(base, ow_c, grids, strides, B, E, H, hd))
        assert_close(got, _port_fp32(base, ow_c, grids, strides, B, E, H, hd), GATE_S32, f"{name} vs the fp32 port")


@pytest.mark.parametrize("what", ["P3", "L5", "hd36", "hd6", "value_ld", "value_misaligned"])
def test_ms_deform_attn_rejects(cuda, what):
    """all checked on the host before anything is enqueued: P != 4 is unsupported (-2), the rest are invalid (-1)"""
    grids, strides, E, H, B, P = [(3, 5, 2), (6, 10, 4)], (8, 4), 64, 2, 1, 4
    if what == "L5":
        grids, strides = grids + [(1, 1, 1), (2, 2, 1), (4, 4, 2)], (32, 16, 8, 4, 2)
    elif what == "hd36":
        E, H = 288, 8
    elif what == "hd6":
        E, H = 96, 16
    rows = B * sum(x * y * z for x, y, z in grids)
    hd = E // H
    value = torch.randn(rows, E, device=cuda)
    ow = torch.randn(rows, H * len(grids) * 4 * 4, device=cuda)
    out = sentinel(rows, E, cuda)
    ld, v = hd, value
    if what == "P3":
        P = 3
    elif what == "value_ld":
        ld = hd
        value = torch.randn(rows, E - 4, device=cuda)
        v = value
    elif what == "value_misaligned":
        v = misaligned(value)
    rc = -2 if what == "P3" else -1
    rejected("occ_ms_deform_attn", v, value.shape[1], ld, ow, out, len(grids), B, _grids(grids), _strides(strides), E,
             H, P, buffers=(out, value, ow), rc=rc)


# ------------------------------------------------------------------------------------------------ occ_neck_token_prep
_COMBOS = [(f, s, p) for f in (0, 1) for s in (0, 1) for p in (0, 1) if f or s or p]


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("L", [1, 3, 4])
@pytest.mark.parametrize("C", [32, 96, 192, 256, 1024])
def test_token_prep_against_fp64(cuda, C, L, B):
    """with and without the LayerNorm; all seven output combinations give the same bits for the outputs present;
    out_s32 = split(out_f32) and out_pos = split(out_f32 + pos[start_l + local]) bit for bit"""
    grids = ref.TOKEN_GRIDS[L]
    x, pos = ref.token_input(grids, B, C, ref.case_seed(C, L, B))
    lw, lb = ref.affine(C, ref.case_seed(C))
    x, pos, lw, lb = (t.to(cuda) for t in (x, pos, lw, lb))
    rows = x.shape[0]
    idx = ref.pos_index(grids, B, cuda)
    special = ref.ln_rows(rows)
    for ln in (None, (lw, lb)):
        want, want_pos = ref.token_prep(x.double(), grids, B, ln=None if ln is None else (lw.double(), lb.double()),
                                        pos=pos.double())
        name = f"token_prep C{C} L{L} B{B} {'LN' if ln else 'no LN'}"
        outs = {}
        for f, s, p in _COMBOS:
            o = [sentinel(rows, C, cuda) if w else None for w in (f, s, p)]
            n = launches("occ_neck_token_prep", x, *(ln or (None, None)), pos if p else None, *o, L, B, _grids(grids),
                         C)
            assert n == 1
            for k, t in enumerate(o):
                if t is None:
                    continue
                if k in outs:
                    same_bits(t, outs[k], f"{name}: output {k} with outputs {(f, s, p)}")
                else:
                    outs[k] = t
        f32, s32, ps = outs[0], outs[1], outs[2]
        assert_close(f32, want, GATE, name)
        if special:
            big = slice(special[2], special[2] + 1)
            assert_close(f32[big], want[big], GATE, f"{name}: row offset by 1e3 x its spread")
            low = slice(special[0], special[0] + 1)
            assert_close(f32[low], want[low], GATE, f"{name}: row with variance near 1e-4")
        if ln is None:
            same_bits(f32, x, f"{name}: out_f32 without the LayerNorm is the input")
        same_bits(s32, ops.to_split(f32), f"{name}: S32 output vs the split of the fp32 output")
        same_bits(ps, ops.to_split(f32 + pos[idx]), f"{name}: out_pos vs split(out_f32 + pos[start_l + local])")
        assert_close(ops.unsplit_weight(ps), want_pos, GATE_S32, f"{name} x + pos (S32)")


@pytest.mark.parametrize("what", ["C160", "ln_w_without_ln_b", "out_pos_without_pos"])
def test_token_prep_rejects(cuda, what):
    grids, B = ref.TOKEN_GRIDS[3], 1
    C = 160 if what == "C160" else 96
    rows = B * sum(x * y * z for x, y, z in grids)
    x, pos = torch.randn(rows, C, device=cuda), torch.randn(rows, C, device=cuda)
    w, b = torch.ones(C, device=cuda), torch.zeros(C, device=cuda)
    outs = [sentinel(rows, C, cuda) for _ in range(3)]
    if what == "ln_w_without_ln_b":
        b = None
    if what == "out_pos_without_pos":
        pos = None
    rejected("occ_neck_token_prep", x, w, b, pos, *outs, len(grids), B, _grids(grids), C, buffers=outs,
             rc=-2 if what == "C160" else -1)


# ------------------------------------------------------------------------------------------------ occ_gn_upsample_add
def _gn_up_case(case, device):
    B, (X, Y, Z), (Xc, Yc, Zc), C, groups = ref.GN_UP_CASES[case]
    cur = ref.gn_input(B, X * Y * Z, C, groups, ref.case_seed(case, 1)).to(device)
    gw, gb = (t.to(device) for t in ref.affine(C, ref.case_seed(C, groups)))
    coarse = ref.coarse_input(B, Xc, Yc, Zc, C, ref.case_seed(case, 2)).to(device)
    return cur.view(B, X, Y, Z, C), gw, gb, coarse


def _gn_up(cur, st, gw, gb, groups, coarse):
    B, X, Y, Z, C = cur.shape
    _, Xc, Yc, Zc, _ = coarse.shape
    out = sentinel(B * X * Y * Z, C, cur.device).view(cur.shape)
    n = launches("occ_gn_upsample_add", cur, st, gw, gb, groups, coarse, out, B, X, Y, Z, Xc, Yc, Zc, C)
    assert n == 1
    return out


@pytest.mark.parametrize("case", range(len(ref.GN_UP_CASES)),
                         ids=lambda i: "B{}-{}x{}x{}-from-{}x{}x{}-C{}-g{}".format(
                             ref.GN_UP_CASES[i][0], *ref.GN_UP_CASES[i][1], *ref.GN_UP_CASES[i][2],
                             *ref.GN_UP_CASES[i][3:]))
def test_gn_upsample_add_against_fp64(cuda, case):
    """the statistics are fp64 sums of the fp32 input (not occ_gn_stats); the planted groups with mean / std = 100 are
    also checked on their own"""
    cur, gw, gb, coarse = _gn_up_case(case, cuda)
    B, X, Y, Z, C = cur.shape
    groups = ref.GN_UP_CASES[case][4]
    st = ref.gn_stats(cur.view(-1, C), B, groups)
    want = ref.gn_upsample_add(cur.double(), st, gw.double(), gb.double(), groups, coarse.double())
    name = f"gn_upsample_add B{B} {X}x{Y}x{Z} from {tuple(coarse.shape[1:4])} C{C} g{groups}"
    out = _gn_up(cur, st, gw, gb, groups, coarse)
    got = ops.unsplit_weight(out.view(-1, C)).view(cur.shape)
    assert_close(got, want, GATE_S32, f"{name} (S32)")
    cpg = C // groups
    for b, gi in ref.gn_special(B, groups):
        sl = (b, Ellipsis, slice(gi * cpg, (gi + 1) * cpg))
        assert_close(got[sl], want[sl], GATE_S32, f"{name}: sample {b} group {gi} (mean / std = 100)")
    same_bits(_gn_up(cur, st, gw, gb, groups, coarse), out, "repeat launch")


@pytest.mark.parametrize("which", ["cur", "coarse", "out_s"])
def test_gn_upsample_add_rejects_misaligned_tensors(cuda, which):
    """the kernels move float4s: a pointer that is not 16-byte aligned is refused on the host"""
    cur, gw, gb, coarse = _gn_up_case(1, cuda)
    B, X, Y, Z, C = cur.shape
    _, Xc, Yc, Zc, _ = coarse.shape
    st = ref.gn_stats(cur.view(-1, C), B, 32)
    out = sentinel(B * X * Y * Z + 1, C, cuda)
    args = {"cur": cur, "coarse": coarse, "out_s": out}
    args[which] = misaligned(args[which])
    rejected("occ_gn_upsample_add", args["cur"], st, gw, gb, 32, args["coarse"], args["out_s"], B, X, Y, Z, Xc, Yc, Zc,
             C, buffers=(out, cur, coarse))


# ------------------------------------------------------------------------------------------------ occ_gn_stats
@pytest.mark.parametrize("case", range(len(ref.GN_STATS_CASES)),
                         ids=lambda i: "B{}-rows{}-C{}-cpg{}".format(*ref.GN_STATS_CASES[i]))
def test_gn_stats_against_fp64(cuda, case):
    """the mean and variance derived from the statistics, and the tensor normalised with them, against fp64; the planted
    groups with mean / std = 100 also on their own.  The statistics are accumulated (+=) into a buffer that already
    holds values."""
    B, rows, C, cpg = ref.GN_STATS_CASES[case]
    groups = C // cpg
    x = ref.gn_input(B, rows, C, groups, ref.case_seed(B, rows, C, cpg)).to(cuda)
    want_st = ref.gn_stats(x, B, groups)
    prior = torch.randn(B, groups, 2, generator=torch.Generator().manual_seed(case), dtype=torch.float64).to(cuda)
    st = prior.clone()
    assert launches("occ_gn_stats", x, st, B, rows, C, cpg) == 1
    got_st = st - prior
    name = f"gn_stats B{B} rows{rows} C{C} cpg{cpg}"
    n = rows * cpg

    def moments(s):
        m = s[..., 0] / n
        return m, s[..., 1] / n - m * m

    (gm, gv), (wm, wv) = moments(got_st), moments(want_st)
    assert_close(gm, wm, GATE, f"{name}: group means")
    assert_close(gv, wv, GATE, f"{name}: group variances")
    one, zero = torch.ones(C, dtype=torch.float64, device=cuda), torch.zeros(C, dtype=torch.float64, device=cuda)
    xd = x.double()
    got = ref.group_norm(xd, got_st, one, zero, rows, groups).view(B, rows, C)
    want = ref.group_norm(xd, want_st, one, zero, rows, groups).view(B, rows, C)
    assert_close(got, want, GATE, f"{name}: normalised tensor")
    for b, gi in ref.gn_special(B, groups):
        sl = (b, slice(None), slice(gi * cpg, (gi + 1) * cpg))
        assert_close(got[sl], want[sl], GATE, f"{name}: normalised sample {b} group {gi} (mean / std = 100)")
        assert_close(gv[b, gi], wv[b, gi], GATE, f"{name}: variance of sample {b} group {gi}")


@pytest.mark.parametrize("what", ["97_groups", "C_not_multiple_of_4", "cpg_not_dividing_C", "x_misaligned"])
def test_gn_stats_rejects(cuda, what):
    B, rows, C, cpg = 1, 8, 96, 3
    if what == "97_groups":
        C, cpg = 97 * 4, 4
    elif what == "C_not_multiple_of_4":
        C, cpg = 98, 2
    elif what == "cpg_not_dividing_C":
        cpg = 5
    x = torch.randn(B * rows, C, device=cuda)
    st = torch.zeros(B, max(1, C // cpg), 2, dtype=torch.float64, device=cuda)
    rejected("occ_gn_stats", misaligned(x) if what == "x_misaligned" else x, st, B, rows, C, cpg, buffers=(st,))
