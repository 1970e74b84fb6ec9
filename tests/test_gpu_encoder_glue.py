"""The dual-path encoder block's glue kernels (csrc/encoder_ops.cu) one launch at a time against the fp64 reference of
tests/encoder_ref.py: occ_gn_relu_zmean_ln (token order and window layout), occ_layernorm (vectorised and generic),
occ_gn_apply, occ_aspp_gap_branch, occ_depthnet_gap_branch and occ_dualpath_fuse.

GroupNorm statistics are computed in fp64 from the same fp32 inputs, so no convolution error enters.  Every case also
checks what the full-block tests cannot see: the launch count of the entry point, bit-identical repeat launches (all
but occ_aspp_gap_branch, whose column sums are fp64 atomics), S32 outputs that are bit for bit the split of the fp32
output, and sentinel bits in every row and column of a sliced or window-layout output that the launch must not write.
tests/test_cpu_encoder_reference.py checks the reference, and that these inputs tell planted mistakes apart.

Gates (tests/util.assert_close, both criteria): GATE for fp32 outputs, GATE_S32 for decoded S32 outputs, for every row,
including the occ_layernorm row offset by 1e3 x its spread (the kernels sum the row shifted by its first element)."""
import pytest
import torch

import encoder_ref as ref
from oracle import port
from util import assert_close, launches, rejected, same_bits, sentinel, untouched
from occformer_b200 import ops

pytestmark = pytest.mark.gpu

GATE, GATE_S32 = ref.GATE_F32, ref.GATE_S32


def _dev(cuda, *ts):
    return [t.to(cuda) for t in ts]


def _d(*ts):
    return [t.double() for t in ts]


# ------------------------------------------------------------------------------------------------ occ_gn_relu_zmean_ln
ZMEAN_CASES = [
    (1, 7, 5, 8, 128, 32),    # R = 4; 35 columns, the last CTA partial
    (2, 7, 5, 8, 128, 32),    # a CTA holds columns of both samples
    (2, 9, 16, 2, 128, 32),   # R = 1 at C = 128
    (1, 10, 6, 3, 128, 16),   # odd Z, 5 columns per CTA, cpg 8
    (2, 5, 7, 1, 128, 32),    # Z = 1: the BEV token is the voxel token
    (1, 9, 8, 16, 128, 32),   # the model's stage-0 depth
    (2, 6, 5, 8, 256, 32),
    (1, 5, 5, 4, 512, 32),
    (2, 4, 4, 2, 1024, 32),
    (1, 3, 3, 12, 1024, 8),   # the Z-column buffer is exactly 48 KiB
]


@pytest.mark.parametrize("B,X,Y,Z,C,groups", ZMEAN_CASES)
def test_gn_relu_zmean_ln_against_fp64(cuda, B, X, Y, Z, C, groups):
    XY = X * Y
    nvox, rows = B * XY * Z, B * XY * (Z + 1)
    y, gw, gb = ref.gn_case(B, XY * Z, C, groups)
    lw, lb = ref.affine(C, ref.case_seed(C, groups, 1))
    y, gw, gb, lw, lb = _dev(cuda, y, gw, gb, lw, lb)
    st = ref.gn_stats(y.double(), B, groups)
    want_tok, want_tokn = ref.gn_relu_zmean_ln(*_d(y), st, *_d(gw, gb, lw, lb), B, XY, Z, groups)

    def run(win_shift, tokn_rows):
        tok, tokn = sentinel(rows, C, cuda), sentinel(tokn_rows, C, cuda)
        n = launches("occ_gn_relu_zmean_ln", y, st, gw, gb, lw, lb, tok, tokn, B, XY, Z, C, groups, X, win_shift)
        assert n == 1
        return tok, tokn

    case = f"B{B} X{X} Y{Y} Z{Z} C{C} g{groups}"
    tok, tokn = run(-1, rows)
    assert_close(tok[:nvox], want_tok[:nvox], GATE, f"gn_relu_zmean_ln {case} tok voxel rows")
    assert_close(tok[nvox:], want_tok[nvox:], GATE, f"gn_relu_zmean_ln {case} tok BEV rows")
    assert_close(ops.unsplit_weight(tokn), want_tokn, GATE_S32, f"gn_relu_zmean_ln {case} tokn (S32)")
    if Z == 1:
        same_bits(tok[nvox:], tok[:nvox], "Z = 1: BEV rows vs voxel rows")
    tok2, tokn2 = run(-1, rows)
    same_bits(tok2, tok, "repeat launch, tok")
    same_bits(tokn2, tokn, "repeat launch, tokn")
    if C == 128:
        wl_rows = ops.lib().occ_window_layout_rows(B, X, Y, Z)
        for shift in (0, 1):
            tok_w, wl = run(shift, wl_rows)
            idx = ops.window_layout_index(B, X, Y, Z, shift).to(cuda)
            same_bits(tok_w, tok, f"win_shift {shift}: tok")
            same_bits(wl[idx], tokn, f"win_shift {shift}: window-layout rows vs token order")
            pad = torch.ones(wl_rows, dtype=torch.bool, device=cuda)
            pad[idx] = False
            untouched(wl[pad], f"win_shift {shift}: pad rows of the window layout")


@pytest.mark.parametrize("Z,C,groups", [(17, 128, 32), (4, 384, 32), (4, 128, 64), (13, 1024, 32)])
def test_gn_relu_zmean_ln_rejects_unsupported_shapes(cuda, Z, C, groups):
    B, X, Y = 1, 3, 3
    XY, rows = X * Y, B * X * Y * (Z + 1)
    y = torch.randn(B * XY * Z, C, device=cuda)
    st = ref.gn_stats(y.double(), B, groups)
    w, b = torch.ones(C, device=cuda), torch.zeros(C, device=cuda)
    tok, tokn = sentinel(rows, C, cuda), sentinel(rows, C, cuda)
    rejected("occ_gn_relu_zmean_ln", y, st, w, b, w, b, tok, tokn, B, XY, Z, C, groups, X, -1, buffers=(tok, tokn))
    untouched(tok, "tok")
    untouched(tokn, "tokn")


# ------------------------------------------------------------------------------------------------ occ_layernorm
@pytest.mark.parametrize("rows", [1, 7, 8, 1001])
@pytest.mark.parametrize("C", [128, 256, 512, 1024, 96, 192, 384, 100])
def test_layernorm_against_fp64(cuda, C, rows):
    """C in {128, 256, 512, 1024}: the vectorised kernel; else the generic one (C = 100: lanes with different trip counts,
    fp32 output only).  Eight rows per CTA: 7 and 1001 leave the last CTA partial."""
    x, w, b = _dev(cuda, ref.ln_input(rows, C, ref.case_seed(rows, C)), *ref.affine(C, ref.case_seed(C)))
    want = ref.layernorm(*_d(x, w, b))

    def run(split):
        out = sentinel(rows, C, cuda)
        assert launches("occ_layernorm", x, w, b, out, rows, C, split) == 1
        return out

    case = f"C{C} rows{rows}"
    out = run(0)
    assert_close(out, want, GATE, f"layernorm {case}")
    special = ref.ln_rows(rows)
    if special:  # the offset row alone: against its own spread, not the largest value of the tensor
        big = slice(special[2], special[2] + 1)
        assert_close(out[big], want[big], GATE, f"layernorm {case} row offset by 1e3 x its spread")
    same_bits(run(0), out, "repeat launch")
    if C % 32 == 0:
        s = run(1)
        same_bits(s, ops.to_split(out), "S32 output vs the split of the fp32 output")
        assert_close(ops.unsplit_weight(s), want, GATE_S32, f"layernorm {case} S32")
        same_bits(run(1), s, "repeat launch, S32")


# ------------------------------------------------------------------------------------------------ occ_gn_apply
# (B, rows_per_batch, C, groups, residual, relu, fp32 output, S32 row pitch, S32 column offsets)
GN_APPLY_CASES = [
    (2, 2500, 32, 32, False, True, True, 160, (0, 32, 64, 96, 128)),  # cpg 1, the ASPP input conv
    (2, 2500, 128, 64, False, True, False, 160, (0, 32)),             # the merged branches into the concat buffer
    (1, 625, 64, 32, True, True, False, 160, (32, 64, 96)),           # bn1 + residual, S32 only
    (1, 49, 1024, 32, True, True, True, 0, ()),                       # output_conv + residual, fp32
    (1, 20000, 192, 32, False, False, True, 256, (32,)),              # the neck: no ReLU, 5 row lanes, 16 idle threads
    (2, 100003, 192, 32, False, True, True, 192, (0,)),               # k > 1 units per CTA, partial CTA per sample
    (3, 300, 1536, 48, False, True, True, 1600, (32,)),               # two column passes, the second part-full
    (2, 77, 40, 10, False, True, True, 0, ()),                        # C not a multiple of 32
]


@pytest.mark.parametrize("case", GN_APPLY_CASES, ids=lambda c: "B{}-rows{}-C{}-g{}".format(*c[:4]))
def test_gn_apply_against_fp64(cuda, case):
    B, rpb, C, groups, with_res, relu, want_f32, ldo, offs = case
    rows = B * rpb
    x, w, b = _dev(cuda, *ref.gn_case(B, rpb, C, groups))
    res = None
    if with_res:
        res = torch.randn(rows, C, generator=torch.Generator().manual_seed(ref.case_seed(*case[:4]))).to(cuda)
    st = ref.gn_stats(x.double(), B, groups)
    want = ref.gn_apply(*_d(x), st, *_d(w, b), rpb, groups, residual=None if res is None else res.double(), relu=relu)

    def run(off):
        out = sentinel(rows, C, cuda) if want_f32 else None
        cat = sentinel(rows, ldo, cuda) if off is not None else None
        n = launches("occ_gn_apply", x, st, w, b, res, out, cat, rows, rpb, C, groups, ldo if cat is not None else C,
                     off or 0, int(relu))
        assert n == 1
        return out, cat

    name = f"gn_apply B{B} rows{rpb} C{C} g{groups}"
    for i, off in enumerate(offs or (None,)):
        out, cat = run(off)
        if out is not None:
            assert_close(out, want, GATE, name)
        if cat is not None:
            sl = cat[:, off:off + C]
            assert_close(ops.unsplit_weight(sl), want, GATE_S32, f"{name} S32 at column {off} of {ldo}")
            untouched(cat[:, :off], f"columns before {off}")
            untouched(cat[:, off + C:], f"columns after {off + C}")
            if out is not None:
                same_bits(sl, ops.to_split(out), "S32 output vs the split of the fp32 output")
        if i == 0:
            out2, cat2 = run(off)
            for a, a2 in ((out, out2), (cat, cat2)):
                if a is not None:
                    same_bits(a2, a, "repeat launch")


# ------------------------------------------------------------------------------------------------ occ_aspp_gap_branch
def _gap_ws(B, ch, device):
    return torch.empty((B, ch * 3 // 2 + 2), dtype=torch.float64, device=device)  # B*ch doubles + B*ch floats


@pytest.mark.parametrize("B,rpb,ch", [(2, 2500, 32), (1, 625, 64), (3, 169, 128), (1, 49, 256), (2, 1, 32)])
def test_aspp_gap_branch_against_fp64(cuda, B, rpb, ch):
    """groups by the model's inner-group rule (BottleNeckASPP of a C = 4 ch block); written at column 4 ch of a 5 ch wide
    concat buffer (the model's slot) and at column 0"""
    groups = port.aspp_groups(4 * ch)
    x, wconv, gw, gb = _dev(cuda, *ref.gap_case(B, rpb, ch, groups))
    want = ref.aspp_gap_branch(*_d(x, wconv, gw, gb), B, groups)
    rows, ldo = B * rpb, 5 * ch
    for off in (4 * ch, 0):
        cat = sentinel(rows, ldo, cuda)
        n = launches("occ_aspp_gap_branch", x, _gap_ws(B, ch, cuda), wconv, gw, gb, cat, B, rpb, ch, groups, ldo, off)
        assert n == 4  # memset, column sums, branch, broadcast
        sl = cat[:, off:off + ch]
        assert_close(ops.unsplit_weight(sl), want, GATE_S32,
                     f"aspp_gap_branch B{B} rows{rpb} ch{ch} g{groups} at column {off}")
        per_sample = sl.contiguous().view(B, rpb, ch)
        same_bits(per_sample, per_sample[:, :1].expand_as(per_sample), "rows of one sample")
        untouched(cat[:, :off], f"columns before {off}")
        untouched(cat[:, off + ch:], f"columns after {off + ch}")


def test_aspp_gap_branch_rejects_a_slice_past_the_row(cuda):
    """out_off + ch > ldo.  The buffer has one spare row, so a library without the check would still write only inside
    the allocation (columns 32..95 of each 64-float row spill into the next row)"""
    B, rpb, ch, groups = 1, 4, 64, 32
    x, wconv, gw, gb = _dev(cuda, *ref.gap_case(B, rpb, ch, groups))
    cat = sentinel(B * rpb + 1, 64, cuda)
    rejected("occ_aspp_gap_branch", x, _gap_ws(B, ch, cuda), wconv, gw, gb, cat, B, rpb, ch, groups, 64, 32,
             buffers=(cat,))
    untouched(cat, "concat buffer")


def test_aspp_gap_branch_rejects_more_than_65535_samples(cuda):
    B, rpb, ch, groups = 65536, 1, 32, 16
    x = torch.randn(B * rpb, ch, device=cuda)
    wconv, gw, gb = torch.randn(ch, ch, device=cuda), torch.ones(ch, device=cuda), torch.zeros(ch, device=cuda)
    cat = sentinel(B * rpb, 5 * ch, cuda)
    rejected("occ_aspp_gap_branch", x, _gap_ws(B, ch, cuda), wconv, gw, gb, cat, B, rpb, ch, groups, 5 * ch, 4 * ch,
             buffers=(cat,))


# ------------------------------------------------------------------------------------------------ occ_depthnet_gap_branch
@pytest.mark.parametrize("B,rpb,ch", [(6, 704, 128), (2, 17, 1024), (1, 1, 32)])
def test_depthnet_gap_branch_against_fp64(cuda, B, rpb, ch):
    """written at column 32 of a ch + 64 wide buffer: live columns on both sides"""
    g = torch.Generator().manual_seed(ref.case_seed(B, rpb, ch))
    w, b = torch.randn(ch, ch, generator=g) * ch ** -0.5, 0.1 * torch.randn(ch, generator=g)
    x, w, b = _dev(cuda, ref.gn_input(B, rpb, ch, 32, ref.case_seed(B, rpb, ch, 32)), w, b)
    want = ref.depthnet_gap_branch(*_d(x, w, b), B)
    rows, ldo, off = B * rpb, ch + 64, 32

    def run():
        cat = sentinel(rows, ldo, cuda)
        ws = torch.empty((2, B, ch), dtype=torch.float32, device=cuda)
        assert launches("occ_depthnet_gap_branch", x, ws, w, b, cat, B, rpb, ch, ldo, off) == 3
        return cat

    cat = run()
    sl = cat[:, off:off + ch]
    assert_close(ops.unsplit_weight(sl), want, GATE_S32, f"depthnet_gap_branch B{B} rows{rpb} ch{ch}")
    per_sample = sl.contiguous().view(B, rpb, ch)
    same_bits(per_sample, per_sample[:, :1].expand_as(per_sample), "rows of one image")
    untouched(cat[:, :off], "columns before the slice")
    untouched(cat[:, off + ch:], "columns after the slice")
    same_bits(run(), cat, "repeat launch (fixed-order sums)")


# ------------------------------------------------------------------------------------------------ occ_dualpath_fuse
def _fuse(cuda, x, bev, cw, cbias, identity, split, st, gw, gb, f32, s32, B, XY, Z, C):
    rows = B * XY * Z
    out = sentinel(rows, C, cuda) if f32 else None
    out_s = sentinel(rows, C, cuda) if s32 else None
    n = launches("occ_dualpath_fuse", x, bev, cw, cbias, identity, split, st, gw if st is not None else None,
                 gb if st is not None else None, 32 if st is not None else 0, out, out_s, B, XY, Z, C)
    assert n == 1
    return out, out_s


@pytest.mark.parametrize("B,XY,Z", [(2, 35, 3), (1, 12, 1)])
@pytest.mark.parametrize("C", [128, 256, 512, 1024])
def test_dualpath_fuse_against_fp64(cuda, C, B, XY, Z):
    """every identity kind (S32 block input, fp32, fp32 GroupNorm'd with id_stats) with fp32-only, S32-only and both
    outputs.  (2, 35, 3): 105 rows per sample, so at R = 2 a warp's two rows belong to different samples, and 210 rows
    is not a multiple of 8R."""
    x, bev, cw, idn = _dev(cuda, *ref.fuse_case(B, XY, Z, C))
    gw, gb = _dev(cuda, *ref.affine(C, ref.case_seed(C, 32)))
    cbias = float(torch.tensor(0.1, dtype=torch.float32))  # the value the kernel receives
    st = ref.gn_stats(idn.double(), B, 32)
    idn_s = ops.to_split(idn)
    kinds = {"S32": (idn_s, 1, None, ops.unsplit_weight(idn_s)), "fp32": (idn, 0, None, idn),
             "fp32+id_stats": (idn, 0, st, idn)}
    for kind, (ident, split, stats, ident_ref) in kinds.items():
        want = ref.dualpath_fuse(*_d(x, bev, cw), cbias, ident_ref.double(), B, XY, Z, id_stats=stats,
                                 id_w=gw.double(), id_b=gb.double(), groups=32)
        name = f"dualpath_fuse C{C} B{B} XY{XY} Z{Z} identity {kind}"
        args = (cuda, x, bev, cw, cbias, ident, split, stats, gw, gb)
        for f32, s32 in ((1, 0), (0, 1), (1, 1)):
            out, out_s = _fuse(*args, f32, s32, B, XY, Z, C)
            if out is not None:
                assert_close(out, want, GATE, name)
            if out_s is not None:
                assert_close(ops.unsplit_weight(out_s), want, GATE_S32, f"{name} S32")
        same_bits(out_s, ops.to_split(out), "S32 output vs the split of the fp32 output")
        out2, out_s2 = _fuse(*args, 1, 1, B, XY, Z, C)
        same_bits(out2, out, "repeat launch")
        same_bits(out_s2, out_s, "repeat launch, S32")


@pytest.mark.parametrize("cbias", [80.0, -80.0])
@pytest.mark.parametrize("C", [128, 256, 512, 1024])
def test_dualpath_fuse_saturated_coefficient(cuda, C, cbias):
    """<x, w> spans +-50 around a bias of +-80: the result stays finite, and where the fp32 sigmoid saturates (z > 20:
    exp(-z) vanishes next to 1; z < -90: exp(-z) overflows) the coefficient is exactly 1 or 0"""
    B, XY, Z = 2, 35, 3
    rows = B * XY * Z
    x, bev, cw, idn = (t.double() for t in ref.fuse_case(B, XY, Z, C))
    target = torch.linspace(-50, 50, rows, dtype=torch.float64)
    x = x + ((target - x @ cw) / (cw @ cw))[:, None] * cw  # <x, cw> = target
    x, bev, cw, idn = _dev(cuda, *(t.float() for t in (x, bev, cw, idn)))
    z = x.double() @ cw.double() + cbias
    want = ref.dualpath_fuse(*_d(x, bev, cw), cbias, idn.double(), B, XY, Z)
    out, out_s = _fuse(cuda, x, bev, cw, cbias, idn, 0, None, None, None, 1, 1, B, XY, Z, C)
    assert bool(torch.isfinite(out).all())
    assert_close(out, want, GATE, f"dualpath_fuse C{C} saturated, bias {cbias:+.0f}")
    same_bits(out_s, ops.to_split(out), "S32 output vs the split of the fp32 output")
    col = torch.arange(rows, device=cuda) // Z
    one, zero = z > 20, z < -90
    assert int(one.sum() if cbias > 0 else zero.sum()) >= rows // 3
    same_bits(out[one], (x + bev[col] + idn)[one], "coefficient exactly 1")
    same_bits(out[zero], (x + idn)[zero], "coefficient exactly 0")
