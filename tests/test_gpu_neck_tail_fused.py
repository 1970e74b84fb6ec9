"""occ_neck_layer_tail (csrc/neck_tail_fused.cu): the pixel decoder's encoder layer after the deformable gather --
output_proj + residual, norms[0], FFN + residual, norms[1] -- as one launch, against an fp64 restatement kept here.

Cases: the nusc_200 pyramid (25x25x2, 50x50x4, 100x100x8 = 91 250 tokens per sample) at B = 1 and B = 4 at the reference
width (E = 192, F = 768), and small pyramids whose row counts leave a ragged last 128-row tile, at E = 192 and at the
E = 96 / F = 192 width of the small neck fixture.  Every case checks all seven output combinations (bit-identical across
combinations), S32 outputs that are bit for bit the split of the fp32 output (and of fp32 output + pos), bit-identical
repeats, one library launch per call, the same bits from a CUDA-graph replay, the single-pass bf16 mode, and a row
offset by 1e3 x its spread (x input of ln_input, its att row zeroed so that the offset reaches norms[0] unchanged)."""
import pytest
import torch

import neck_ref as ref
from util import assert_close, graph_replay, same_bits
from occformer_b200 import ops

pytestmark = pytest.mark.gpu

GATE = 5e-5        # fp32 outputs and decoded S32 outputs vs fp64 (four chained contractions and two LayerNorms)
GATE_BF16 = 3e-2   # single-pass bf16 mode vs fp64
NUSC_200 = [(25, 25, 2), (50, 50, 4), (100, 100, 8)]
# (grids, B, E, F)
CASES = {
    "nusc200_B1": (NUSC_200, 1, 192, 768),
    "nusc200_B4": (NUSC_200, 4, 192, 768),
    "ragged_L3_B3": (ref.TOKEN_GRIDS[3], 3, 192, 768),
    "ragged_L4_B1": (ref.TOKEN_GRIDS[4], 1, 192, 768),
    "E96_L3_B2": (ref.TOKEN_GRIDS[3], 2, 96, 192),
}
_COMBOS = [(f, s, p) for f in (0, 1) for s in (0, 1) for p in (0, 1) if f or s or p]


def _layer_norm(y, w, b, eps=ref.EPS):
    m = y.mean(-1, keepdim=True)
    var = ((y - m) ** 2).mean(-1, keepdim=True)
    return (y - m) * (var + eps).rsqrt() * w + b


def tail_ref(att, x, wo, bo, ln1, w1, b1, w2, b2, ln2, pos_rows):
    """fp64: out = LN2(x1 + ReLU(x1 w1^T + b1) w2^T + b2), x1 = LN1(x + att wo^T + bo); -> (out, out + pos_rows).
    att and the weights are the values their S32 form holds (decoded)."""
    d = lambda t: t.double()  # noqa: E731
    x1 = _layer_norm(d(x) + d(att) @ d(wo).T + d(bo), d(ln1[0]), d(ln1[1]))
    y2 = x1 + torch.relu(x1 @ d(w1).T + d(b1)) @ d(w2).T + d(b2)
    out = _layer_norm(y2, d(ln2[0]), d(ln2[1]))
    return out, out + d(pos_rows)


def _case(name, device):
    """inputs of a case: S32 operands (att, wo, w1, w2) plus their decoded values, the rest fp32"""
    grids, B, E, F = CASES[name]
    seed = ref.case_seed(len(grids), B, E, F)
    x, pos = ref.token_input(grids, B, E, seed)
    rows = x.shape[0]
    g = torch.Generator().manual_seed(seed + 7)
    rn = lambda *s, std=1.0: (std * torch.randn(*s, generator=g)).float()  # noqa: E731
    att = rn(rows, E)
    special = ref.ln_rows(rows)
    if special:
        att[special[2]] = 0.0  # the offset row of ln_input reaches norms[0] as x + bo
    wo, w1, w2 = rn(E, E, std=E ** -0.5), rn(F, E, std=E ** -0.5), rn(E, F, std=F ** -0.5)
    bo, b1, b2 = 0.1 * rn(E), 0.1 * rn(F), 0.1 * rn(E)
    ln1, ln2 = ref.affine(E, seed + 1), ref.affine(E, seed + 2)
    c = dict(grids=grids, B=B, E=E, F=F, rows=rows, special=special,
             x=x.to(device), pos=pos.to(device), bo=bo.to(device), b1=b1.to(device), b2=b2.to(device),
             ln1=tuple(t.to(device) for t in ln1), ln2=tuple(t.to(device) for t in ln2))
    c["att_s"] = ops.to_split(att.to(device))
    for k, w in (("wo", wo), ("w1", w1), ("w2", w2)):
        c[k + "_s"] = ops.split_weight(w.to(device))
    c["pos_rows"] = c["pos"][ref.pos_index(grids, B, device)]
    return c


def _run(c, want_f32=True, want_s32=True, want_pos=True):
    """one call of ops.neck_layer_tail -> (outputs, library launches it enqueued)"""
    n0 = ops.LAUNCH_COUNT[0]
    out = ops.neck_layer_tail(c["att_s"], c["x"], c["wo_s"], c["bo"], c["ln1"], c["w1_s"], c["b1"], c["w2_s"], c["b2"],
                              c["ln2"], c["grids"], c["B"], pos=c["pos"], want_f32=want_f32, want_s32=want_s32,
                              want_pos=want_pos)
    return out, ops.LAUNCH_COUNT[0] - n0


def _want(c):
    dec = ops.unsplit_weight
    return tail_ref(dec(c["att_s"]), c["x"], dec(c["wo_s"]), c["bo"], c["ln1"], dec(c["w1_s"]), c["b1"], dec(c["w2_s"]),
                    c["b2"], c["ln2"], c["pos_rows"])


@pytest.mark.parametrize("name", list(CASES))
def test_neck_layer_tail_against_fp64(cuda, name):
    c = _case(name, cuda)
    want, want_pos = _want(c)
    outs = {}
    for combo in _COMBOS:
        o, n = _run(c, *map(bool, combo))
        assert n == 1, f"{name}: {n} launches for one call"
        for k, t in enumerate(o):
            assert (t is None) == (not combo[k])
            if t is None:
                continue
            if k in outs:
                same_bits(t, outs[k], f"{name}: output {k} with outputs {combo}")
            else:
                outs[k] = t
    f32, s32, ps = outs[0], outs[1], outs[2]
    assert_close(f32, want, GATE, f"{name}: out fp32")
    assert_close(ops.unsplit_weight(ps), want_pos, GATE, f"{name}: out + pos (S32)")
    if c["special"]:
        big = slice(c["special"][2], c["special"][2] + 1)
        assert_close(f32[big], want[big], GATE, f"{name}: row offset by 1e3 x its spread")
    same_bits(s32, ops.to_split(f32), f"{name}: S32 output vs the split of the fp32 output")
    same_bits(ps, ops.to_split(f32 + c["pos_rows"]), f"{name}: pos output vs split(out + pos[start_l + local])")
    # repeats and a CUDA-graph replay give the same bits
    again, _ = _run(c)
    for a, b in zip(again, (f32, s32, ps)):
        same_bits(a, b, f"{name}: repeat")
    captured = []
    graph_replay(lambda: captured.extend(_run(c)[0]), captured)
    for a, b in zip(captured, (f32, s32, ps)):
        same_bits(a, b, f"{name}: CUDA-graph replay")


@pytest.mark.parametrize("name", ["nusc200_B1", "E96_L3_B2"])
def test_neck_layer_tail_bf16_mode(cuda, name):
    c = _case(name, cuda)
    want, want_pos = _want(c)
    with ops.precision("bf16"):
        (f32, _, ps), n = _run(c)
    assert n == 1
    assert_close(f32, want, GATE_BF16, f"{name}: bf16 mode out fp32")
    assert_close(ops.unsplit_weight(ps), want_pos, GATE_BF16, f"{name}: bf16 mode out + pos (S32)")


_BAD = ["E160", "F48", "att_rows", "w2_shape", "att_f64", "pos_missing", "rows_vs_grids"]


@pytest.mark.parametrize("what", _BAD)
def test_neck_layer_tail_rejects(cuda, what):
    """bad shapes and dtypes fail on the host: nothing is enqueued"""
    grids, B = ref.TOKEN_GRIDS[3], 1
    E, F = (160, 640) if what == "E160" else (192, 48 if what == "F48" else 768)
    rows = B * sum(x * y * z for x, y, z in grids)
    dev = cuda
    att = torch.randn(rows + (1 if what == "att_rows" else 0), E, device=dev)
    if what == "att_f64":
        att = att.double()
    x = torch.randn(rows + (3 if what == "rows_vs_grids" else 0), E, device=dev)
    if what == "rows_vs_grids":
        att = torch.randn(rows + 3, E, device=dev)
    wo, w1 = torch.randn(E, E, device=dev), torch.randn(F, E, device=dev)
    w2 = torch.randn(E, F + (32 if what == "w2_shape" else 0), device=dev)
    v = lambda n: torch.randn(n, device=dev)  # noqa: E731
    pos = None if what == "pos_missing" else torch.randn(rows, E, device=dev)
    n0 = ops.LAUNCH_COUNT[0]
    with pytest.raises((AssertionError, RuntimeError)):
        ops.neck_layer_tail(att, x, wo, v(E), (v(E), v(E)), w1, v(F), w2, v(E), (v(E), v(E)), grids, B, pos=pos,
                            want_pos=True)
    torch.cuda.synchronize()
    assert ops.LAUNCH_COUNT[0] == n0, f"{what}: enqueued work before rejecting the call"
