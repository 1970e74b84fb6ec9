"""The Swin attention and block-tail kernels one launch at a time against the fp64 reference of tests/swin_ref.py:
occ_window_attention (csrc/window_attn.cu, the C = 256 / 512 / 1024 stages), occ_swin_qkv_attention (csrc/
swin_attn_fused.cu, QKV projection + attention, C = 128) and occ_swin_proj_ffn (csrc/swin_mlp_fused.cu, the C = 128
tail).  tests/test_cpu_swin_reference.py checks the reference, and that these inputs tell planted mistakes apart.

Geometry: every residue of X and Y mod 7 with the shift on and off, X, Y < 7, B = 1, 2, 3; an odd window count (the
last window pair holds a phantom window); the model's stage shapes at B = 1, each running more than WA_STAGES units per
CTA so the loader ring wraps.  Each launch is also checked for what the block tests cannot see: one launch per call,
bit-identical repeats and CUDA-graph replay, NaN sentinel rows past the output, head-major vs reference qkv order,
MMA padding rows of the window layout, single-pass bf16 mode, and argument rejection with nothing enqueued.

Gates (tests/util.assert_close, both criteria): GATE = 5e-5 for every output (attention outputs decoded from S32), but
  * occ_swin_qkv_attention's allclose criterion is widened element by element by swin_ref.pv_error, 2^-16 sum_j p_j
    |v_j|: the split P V product errs in proportion to the values it averages, and at the stage-0 shape (87 M elements)
    10 to 16 outputs that average values ~10x their own size sit past GATE * (rms + |out|) by that much; rel_max stays
    at GATE;
  * the fused kernel's large-logit window.  The reference takes q / k / v as the attention core consumes them (the
    kernel's fp32 projection split to hi + lo, swin_ref.qkv_attention(split_qkv=True)); what remains is the lo * lo
    product the three passes drop, up to 2^-18 * scale * sum_d |q_d||k_d| per score (swin_ref.qk_split_bound; ~4e-4
    at the planted |q||k| ~ 549), which moves an output by at most twice that times max |v|.  That window's gate is
    GATE plus this bound relative to its largest output;
  * occ_swin_proj_ffn's row offset by 1e3 x its spread, judged on its own: y1 + b2 (~1e3) is rounded to fp32 when it is
    formed (3 roundings), parked, and then accumulated onto by 8 wgmma per pass; each of those 3 + 8 * 3 additions may
    round by one ulp of the row's largest value, and on top of that the FFN part keeps GATE."""
import math

import pytest
import torch

import swin_ref as ref
from util import (assert_close, graph_replay, launches, misaligned, parity_log, rejected, rel_err, same_bits,
                  sentinel, untouched)
from occformer_b200 import ops

pytestmark = pytest.mark.gpu

GATE = ref.GATE
WA_STAGES = 4          # csrc/window_geom.cuh: units in flight per CTA of window_attn_tc_kernel
EXTRA_ROWS = 3         # sentinel rows behind every output


def _sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _units_per_cta(nwin, heads):
    """window pairs of the busiest CTA (both attention kernels: CTA groups of `heads` CTAs, one per SM)"""
    npairs = (nwin + 1) // 2
    groups = min(_sm_count() // heads, npairs)
    return -(-npairs // groups)


def _window_rows(B, X, Y, Z, shift, name, plants, device):
    """token rows of a planted window (real tokens only)"""
    if name not in plants:
        return torch.zeros(0, dtype=torch.long, device=device)
    r = ref.windows(B, X, Y, Z, shift)[0][plants[name]]
    return r[r >= 0].to(device)


# ------------------------------------------------------------------------------------------------ occ_window_attention
def _wa(cuda, B, X, Y, Z, C, shift):
    """-> (run(head_major) -> S32 output slice of a sentinel buffer, fp64 reference, plants)"""
    heads = C // ref.HD
    qkv, b, table, plants = ref.qkv_case(B, X, Y, Z, C, shift, ref.case_seed(B, X, Y, Z))
    qkv_s, b_s = ops.split_weight(qkv.to(cuda)), ops.split_weight(b.view(1, -1).to(cuda)).view(-1)
    bias = ref.bias_pad(table).to(cuda)
    qkv_d, b_d = ops.unsplit_weight(qkv_s).double(), ops.unsplit_weight(b_s.view(1, -1)).view(-1).double()
    want = ref.window_attention(qkv_d, b_d, table.double().to(cuda), B, X, Y, Z, C, heads, shift)
    # head-major order moves whole 32-column S32 chunks: [q|k|v][head] -> [head][q|k|v]
    hm = qkv_s.view(-1, 3, heads, 32).permute(0, 2, 1, 3).reshape(qkv_s.shape[0], 3 * C).contiguous()
    hm_b = b_s.view(3, heads, 32).permute(1, 0, 2).reshape(-1).contiguous()
    rows = qkv.shape[0]

    def run(head_major=False):
        buf = sentinel(rows + EXTRA_ROWS, C, cuda)
        out = buf[:rows]
        a, bb = (hm, hm_b) if head_major else (qkv_s, b_s)
        n = launches("occ_window_attention", a, bb, bias, out, B, X, Y, Z, C, heads, int(shift), int(head_major))
        assert n == 1, f"{n} launches"
        untouched(buf[rows:], "rows past the output")
        return out

    return run, want, plants, (qkv_s, b_s, bias)


@pytest.mark.parametrize("shift", [False, True])
@pytest.mark.parametrize("B,X,Y,Z", ref.RESIDUE_SHAPES + [ref.ODD_SHAPE])
def test_window_attention_geometry(cuda, B, X, Y, Z, shift):
    C = 128
    run, want, plants, _ = _wa(cuda, B, X, Y, Z, C, shift)
    out = run()
    case = f"B{B} {X}x{Y}x{Z} shift={int(shift)} ({ref.n_windows(B, X, Y, Z)} windows)"
    assert_close(ops.unsplit_weight(out), want, GATE, f"window_attention {case}")
    for name in ("large", "onehot", "pad", "uniform"):
        r = _window_rows(B, X, Y, Z, shift, name, plants, cuda)
        if r.numel():
            assert_close(ops.unsplit_weight(out[r]), want[r], GATE, f"window_attention {case} {name} window")
    same_bits(run(), out, "repeat launch")
    same_bits(run(head_major=True), out, "head-major vs reference qkv order")


def _wrap_shapes():
    # (B, X, Y, Z, C): the model's C > 128 stages at B = 1 (100x100x8: 2 025 windows, odd), and for 1, 2 and 4 heads an
    # odd window count with more than WA_STAGES units per CTA on a 132-SM H100
    return [(1, 100, 100, 8, 256), (1, 50, 50, 4, 512), (1, 25, 25, 2, 1024), (1, 49, 49, 22, 32), (1, 49, 49, 10, 64),
            (1, 49, 49, 6, 128)]


@pytest.mark.parametrize("B,X,Y,Z,C", _wrap_shapes())
def test_window_attention_stage_shapes_wrap_the_ring(cuda, B, X, Y, Z, C):
    heads = C // ref.HD
    units = _units_per_cta(ref.n_windows(B, X, Y, Z), heads)
    assert units > WA_STAGES, f"{units} units per CTA at {_sm_count()} SMs: the ring does not wrap"
    for shift in (True, False):
        run, want, _, _ = _wa(cuda, B, X, Y, Z, C, shift)
        out = run()
        assert_close(ops.unsplit_weight(out), want, GATE,
                     f"window_attention C{C} B{B} {X}x{Y}x{Z} shift={int(shift)} ({units} units per CTA)")
        if shift:
            same_bits(run(head_major=True), out, "head-major vs reference qkv order")


def test_window_attention_graph_replay_and_bf16(cuda):
    B, X, Y, Z = ref.ODD_SHAPE
    C = 128
    run, want, _, (qkv_s, b_s, bias) = _wa(cuda, B, X, Y, Z, C, True)
    out = run()
    rows = out.shape[0]
    g_out = torch.empty_like(out)
    graph_replay(lambda: ops._call("occ_window_attention", qkv_s, b_s, bias, g_out, B, X, Y, Z, C, C // 32, 1, 0),
                 [g_out])
    same_bits(g_out, out, "CUDA-graph replay")
    with ops.precision("bf16"):
        low = run()
    assert rows == low.shape[0]
    assert_close(ops.unsplit_weight(low), want, ref.BF16_GATE, "window_attention single-pass bf16")


# ------------------------------------------------------------------------------------------------ occ_swin_qkv_attention
def _fused(cuda, B, X, Y, Z, shift):
    """-> (run(pad_fill=None) -> S32 output slice of a sentinel buffer, fp64 reference, plants, decoded fp64 qkv + bias,
    launch arguments)"""
    C, heads = 128, 4
    tok, w, b, table, plants = ref.token_case(B, X, Y, Z, shift, ref.case_seed(B, X, Y, Z))
    perm = ref.head_major_perm(C, heads).to(cuda)
    tok_s = ops.split_weight(tok.to(cuda))
    w_hm = ops.split_weight(w.to(cuda)[perm])
    b_hm = b.to(cuda)[perm].contiguous()
    w_ref = torch.empty(3 * C, C, dtype=torch.float64, device=cuda)
    w_ref[perm] = ops.unsplit_weight(w_hm).double()
    b_ref = b.double().to(cuda)
    tok_d = ops.unsplit_weight(tok_s).double()
    table_d = table.double().to(cuda)
    want, pv = ref.qkv_attention(tok_d, w_ref, b_ref, table_d, B, X, Y, Z, C, heads, shift, split_qkv=True,
                                 with_abs=True)
    wl = ops.to_window_layout(tok_s, B, X, Y, Z, shift)
    bias = ref.bias_pad(table).to(cuda)
    rows = tok.shape[0]

    def run(tokens=wl):
        buf = sentinel(rows + EXTRA_ROWS, C, cuda)
        out = buf[:rows]
        n = launches("occ_swin_qkv_attention", tokens, w_hm, b_hm, bias, out, B, X, Y, Z, C, heads, int(shift))
        assert n == 1, f"{n} launches"
        untouched(buf[rows:], "rows past the output")
        return out

    return run, want, plants, (ref.s32(tok_d @ w_ref.T + b_ref), ref.s32(b_ref), pv), (wl, w_hm, b_hm, bias)


def _assert_pv_close(got, want, pv, what):
    """assert_close at GATE, the allclose criterion widened element by element by ref.pv_error"""
    rel = rel_err(got, want)
    rms = float(want.pow(2).mean().sqrt())
    nv = int(((got - want).abs() > GATE * rms + GATE * want.abs() + ref.pv_error(pv)).sum())
    parity_log(f"[parity] {what}: rel_max {rel:.2e} allclose_violations {nv}/{got.numel()} (tol {GATE:.0e} + P V split)")
    assert rel <= GATE and nv == 0, f"{what}: rel_max {rel:.3e}, allclose + P V split violations {nv}"


def _judge_fused(out, want, qkv_d, b_d, pv, plants, B, X, Y, Z, shift, case):
    """every row outside the large-logit window at GATE (elements also within ref.pv_error); that window at GATE + its
    lo * lo bound"""
    dev = out.device
    large = _window_rows(B, X, Y, Z, shift, "large", plants, dev)
    rest = torch.ones(out.shape[0], dtype=torch.bool, device=dev)
    rest[large] = False
    got = ops.unsplit_weight(out).double()
    _assert_pv_close(got[rest], want[rest], pv[rest], f"swin_qkv_attention {case}")
    for name in ("onehot", "pad", "uniform"):
        r = _window_rows(B, X, Y, Z, shift, name, plants, dev)
        if r.numel():
            assert_close(got[r], want[r], GATE, f"swin_qkv_attention {case} {name} window")
    if large.numel():
        bound = ref.qk_split_bound(qkv_d, b_d, B, X, Y, Z, 128, 4, shift, plants["large"])
        rr = ref.windows(B, X, Y, Z, shift)[0][plants["large"]].to(dev)
        v = torch.where((rr < 0)[:, None], b_d, qkv_d[rr.clamp_min(0)])[:, 256:]
        gate = GATE + 2 * bound * float(v.abs().max()) / float(want[large].abs().max())
        parity_log(f"[gate] swin_qkv_attention {case} large-logit window: split bound {bound:.2e} per score -> gate "
                   f"{gate:.2e}")
        assert_close(got[large], want[large], gate, f"swin_qkv_attention {case} large-logit window")


@pytest.mark.parametrize("shift", [False, True])
@pytest.mark.parametrize("B,X,Y,Z", ref.RESIDUE_SHAPES + [ref.ODD_SHAPE, (1, 200, 200, 16)])
def test_swin_qkv_attention_geometry(cuda, B, X, Y, Z, shift):
    """(1, 200, 200, 16): the model's stage 0 at B = 1 (14 297 windows: odd)"""
    run, want, plants, (qkv_d, b_d, pv), _ = _fused(cuda, B, X, Y, Z, shift)
    out = run()
    case = f"B{B} {X}x{Y}x{Z} shift={int(shift)} ({ref.n_windows(B, X, Y, Z)} windows)"
    _judge_fused(out, want, qkv_d, b_d, pv, plants, B, X, Y, Z, shift, case)
    same_bits(run(), out, "repeat launch")
    if (B, X, Y, Z) == (1, 200, 200, 16):
        assert _units_per_cta(ref.n_windows(B, X, Y, Z), 4) > 2


@pytest.mark.parametrize("B,X,Y,Z,shift", [ref.MISTAKE_CASE, (*ref.ODD_SHAPE, True), (1, 4, 4, 3, False)])
def test_swin_qkv_attention_ignores_window_padding_rows(cuda, B, X, Y, Z, shift):
    """rows 49..63 of every window (the phantom window's too) hold finite non-zero values: the same bits as zeros"""
    run, _, _, _, (wl, *_rest) = _fused(cuda, B, X, Y, Z, shift)
    out = run()
    filled = wl.clone().view(-1, 64, 128)
    g = torch.Generator(device=wl.device).manual_seed(5)
    pad = torch.randn(filled.shape[0] * 15, 128, generator=g, device=wl.device) * 3 + 1
    filled[:, ref.WT:] = ops.split_weight(pad).view(-1, 15, 128)
    same_bits(run(filled.view_as(wl)), out, "window layout with non-zero MMA padding rows")


def test_swin_qkv_attention_graph_replay_and_bf16(cuda):
    B, X, Y, Z = ref.ODD_SHAPE
    run, want, plants, _, (wl, w_hm, b_hm, bias) = _fused(cuda, B, X, Y, Z, True)
    out = run()
    g_out = torch.empty_like(out)
    graph_replay(lambda: ops._call("occ_swin_qkv_attention", wl, w_hm, b_hm, bias, g_out, B, X, Y, Z, 128, 4, 1),
                 [g_out])
    same_bits(g_out, out, "CUDA-graph replay")
    with ops.precision("bf16"):
        low = run()
    # the large-logit window is left out: a single bf16 pass moves its ~97 scores by ~0.4
    keep = torch.ones(out.shape[0], dtype=torch.bool, device=cuda)
    keep[_window_rows(B, X, Y, Z, True, "large", plants, cuda)] = False
    assert_close(ops.unsplit_weight(low)[keep], want[keep], ref.BF16_GATE, "swin_qkv_attention single-pass bf16")


# ------------------------------------------------------------------------------------------------ occ_swin_proj_ffn
def _tail(cuda, M):
    att, tok, wp, bp, lw, lb, w1, b1, w2, b2 = (t.to(cuda) for t in ref.tail_case(M, ref.case_seed(M)))
    att_s, wp_s, w1_s, w2_s = (ops.split_weight(t) for t in (att, wp, w1, w2))
    att_d, wp_d, w1_d, w2_d = (ops.unsplit_weight(t).double() for t in (att_s, wp_s, w1_s, w2_s))
    want = ref.swin_tail(att_d, tok.double(), wp_d, bp.double(), lw.double(), lb.double(), w1_d, b1.double(), w2_d,
                         b2.double())
    y1 = tok.double() + att_d @ wp_d.T + bp.double()
    args = (att_s, tok, wp_s, bp, lw, lb, w1_s, b1, w2_s, b2)

    def run():
        buf = sentinel(M + EXTRA_ROWS, 128, cuda)
        out = buf[:M]
        n = launches("occ_swin_proj_ffn", *args, out, M, 128)
        assert n == 1, f"{n} launches"
        untouched(buf[M:], "rows past the output")
        return out

    return run, want, y1 + b2.double(), args


@pytest.mark.parametrize("M", [1, 127, 128, 129, 1000, 128 * 132 * 3 + 77, 128 * 132 * 2, 680000])
def test_swin_proj_ffn_against_fp64(cuda, M):
    """M: one row, a partial tile, one tile, one row past it, and the row counts of the existing tail test; 680 000 is
    stage 0 (200 x 200 x 17 tokens) at B = 1"""
    run, want, resid, _ = _tail(cuda, M)
    out = run()
    special = ref.tail_rows(M)
    keep = torch.ones(M, dtype=torch.bool, device=cuda)
    keep[list(special)] = False
    assert_close(out[keep], want[keep], GATE, f"swin_proj_ffn M={M}")
    if special:
        low, const, big = special
        assert_close(out[low:low + 1], want[low:low + 1], GATE, f"swin_proj_ffn M={M} LN2 variance 1e-4 row")
        assert_close(out[const:const + 1], want[const:const + 1], GATE, f"swin_proj_ffn M={M} constant row")
        top = float(want[big].abs().max())
        ulp = 2.0 ** (math.floor(math.log2(top)) - 23)
        ffn = float((want[big] - resid[big]).abs().max())
        allowed = (3 + 8 * 3) * ulp + GATE * ffn
        err = float((out[big].double() - want[big]).abs().max())
        parity_log(f"[parity] swin_proj_ffn M={M} row offset by 1e3: max err {err:.2e} = {err / ulp:.1f} ulp "
                   f"(allowed {allowed:.2e})")
        assert err <= allowed, f"offset row: max error {err:.3e} > {allowed:.3e}"
    same_bits(run(), out, "repeat launch")


def test_swin_proj_ffn_graph_replay_and_bf16(cuda):
    M = ref.TAIL_MISTAKE_M
    run, want, _, args = _tail(cuda, M)
    out = run()
    g_out = torch.empty_like(out)
    graph_replay(lambda: ops._call("occ_swin_proj_ffn", *args, g_out, M, 128), [g_out])
    same_bits(g_out, out, "CUDA-graph replay")
    with ops.precision("bf16"):
        low = run()
    assert_close(low, want, ref.BF16_GATE, "swin_proj_ffn single-pass bf16")


# ------------------------------------------------------------------------------------------------ rejections
def test_window_attention_rejects_bad_arguments(cuda):
    B, X, Y, Z, C, heads = 1, 7, 7, 1, 128, 4
    rows = B * X * Y * (Z + 1)
    qkv, b = torch.zeros(rows, 3 * C, device=cuda), torch.zeros(3 * C, device=cuda)
    bias, out = torch.zeros(heads * 8, ref.BIAS_FLOATS, device=cuda), sentinel(rows, C, cuda)
    name = "occ_window_attention"
    rejected(name, qkv, b, bias, out, B, X, Y, Z, C, 3, 1, 0, buffers=(out,))               # C != heads * 32
    rejected(name, misaligned(qkv), b, bias, out, B, X, Y, Z, C, heads, 1, 0, buffers=(out,))
    rejected(name, qkv, b, bias, misaligned(out), B, X, Y, Z, C, heads, 1, 0, buffers=(out,))
    r0 = B * X * Y
    rejected(name, qkv[:r0], b, bias, out[:r0], B, X, Y, 0, C, heads, 1, 0, buffers=(out,))   # Z = 0
    h = _sm_count() + 1                                                                         # more heads than SMs
    qkv_h, b_h = torch.zeros(rows, 3 * 32 * h, device=cuda), torch.zeros(3 * 32 * h, device=cuda)
    bias_h, out_h = torch.zeros(h, ref.BIAS_FLOATS, device=cuda), sentinel(rows, 32 * h, cuda)
    rejected(name, qkv_h, b_h, bias_h, out_h, B, X, Y, Z, 32 * h, h, 1, 0, buffers=(out_h,))


def test_swin_qkv_attention_rejects_bad_arguments(cuda):
    """(more heads than SMs cannot be asked of it: C = 128 fixes four heads)"""
    B, X, Y, Z, C, heads = 1, 7, 7, 1, 128, 4
    rows = B * X * Y * (Z + 1)
    wl_rows = ops.lib().occ_window_layout_rows(B, X, Y, Z)
    wl, w, b = torch.zeros(wl_rows, C, device=cuda), torch.zeros(3 * C, C, device=cuda), torch.zeros(3 * C, device=cuda)
    bias, out = torch.zeros(8, ref.BIAS_FLOATS, device=cuda), sentinel(rows, C, cuda)
    name = "occ_swin_qkv_attention"
    rejected(name, wl, w, b, bias, out, B, X, Y, Z, C, 3, 1, buffers=(out,))                 # C != heads * 32
    rejected(name, misaligned(wl), w, b, bias, out, B, X, Y, Z, C, heads, 1, buffers=(out,))
    rejected(name, wl, w, b, bias, misaligned(out), B, X, Y, Z, C, heads, 1, buffers=(out,))
    r0 = B * X * Y
    rejected(name, wl, w, b, bias, out[:r0], B, X, Y, 0, C, heads, 1, buffers=(out,))        # Z = 0
    C2 = 256                                                                                   # C != 128: unsupported
    wl2, w2, b2 = torch.zeros(wl_rows, C2, device=cuda), torch.zeros(3 * C2, C2, device=cuda), torch.zeros(3 * C2,
                                                                                                     device=cuda)
    out2 = sentinel(rows, C2, cuda)
    rejected(name, wl2, w2, b2, bias, out2, B, X, Y, Z, C2, 8, 1, buffers=(out2,), rc=-2)


def test_swin_proj_ffn_rejects_bad_arguments(cuda):
    M, C = 200, 128
    att, tok = torch.zeros(M, C, device=cuda), torch.zeros(M, C, device=cuda)
    w, v = torch.zeros(C, C, device=cuda), torch.zeros(C, device=cuda)
    out = sentinel(M, C, cuda)
    name = "occ_swin_proj_ffn"
    rejected(name, att, tok, w, v, v, v, w, v, w, v, out, 0, C, buffers=(out,))  # M = 0
    rejected(name, misaligned(att), tok, w, v, v, v, w, v, w, v, out, M, C, buffers=(out,))
    rejected(name, att, tok, w, v, v, v, w, v, w, v, misaligned(out), M, C, buffers=(out,))
    C2 = 256                                                                                   # C != 128: unsupported
    att2, tok2, w2, v2 = (torch.zeros(M, C2, device=cuda), torch.zeros(M, C2, device=cuda),
                          torch.zeros(C2, C2, device=cuda), torch.zeros(C2, device=cuda))
    out2 = sentinel(M, C2, cuda)
    rejected(name, att2, tok2, w2, v2, v2, v2, w2, v2, w2, v2, out2, M, C2, buffers=(out2,), rc=-2)
