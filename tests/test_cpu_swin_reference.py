"""The fp64 reference of tests/test_gpu_swin_attention.py (tests/swin_ref.py) against oracle.port and against planted
mistakes.  Its per-window gather equals port.shift_window_msa to fp64 round-off at every residue of X and Y mod 7, with
the shift on and off, at B = 1, 2, 3; composed with the block tail it equals port.swin_block; and on the GPU test's own
inputs, each planted mistake moves the result by more than 10x the GPU gate.  A GPU failure then points at a kernel,
and a case that cannot tell a mistake apart fails here."""
import pytest
import torch
import torch.nn.functional as F

import swin_ref as ref
from oracle import port
from util import rel_err

BITE = 10 * ref.GATE


def _images(rows, B, X, Y, Z):
    """token rows -> (B*(Z+1), X*Y, F) images in the library's image order: (b, z) voxel slices, then the BEV images"""
    F_ = rows.shape[1]
    nvox = B * X * Y * Z
    vox = rows[:nvox].view(B, X, Y, Z, F_).permute(0, 3, 1, 2, 4).reshape(B * Z, X * Y, F_)
    return torch.cat([vox, rows[nvox:].view(B, X * Y, F_)])


def _rows(img, B, X, Y, Z):
    """inverse of _images"""
    F_ = img.shape[-1]
    vox = img[:B * Z].view(B, Z, X, Y, F_).permute(0, 2, 3, 1, 4).reshape(-1, F_)
    return torch.cat([vox, img[B * Z:].reshape(-1, F_)])


def _msa_state(w, b, table, C):
    return {"w_msa.qkv.weight": w, "w_msa.qkv.bias": b, "w_msa.proj.weight": torch.eye(C, dtype=torch.float64),
            "w_msa.proj.bias": torch.zeros(C, dtype=torch.float64), "w_msa.relative_position_bias_table": table}


@pytest.mark.parametrize("shift", [False, True])
@pytest.mark.parametrize("B,X,Y,Z", ref.RESIDUE_SHAPES + [ref.ODD_SHAPE, (2, 18, 25, 1)])
def test_window_attention_equals_port(B, X, Y, Z, shift):
    C, heads = 64, 2
    g = torch.Generator().manual_seed(ref.case_seed(B, X, Y, Z))
    rows = B * X * Y * (Z + 1)
    tok = torch.randn(rows, C, generator=g, dtype=torch.float64)
    w = torch.randn(3 * C, C, generator=g, dtype=torch.float64) * C ** -0.5
    b = 0.3 * torch.randn(3 * C, generator=g, dtype=torch.float64)
    table = torch.randn(169, heads, generator=g, dtype=torch.float64)
    want = port.shift_window_msa(_images(tok, B, X, Y, Z), (X, Y), _msa_state(w, b, table, C), "", heads,
                                 3 if shift else 0)
    got = ref.qkv_attention(tok, w, b, table, B, X, Y, Z, C, heads, shift)
    torch.testing.assert_close(got, _rows(want, B, X, Y, Z), rtol=1e-12, atol=1e-12)
    perm = ref.head_major_perm(C, heads)
    hm = ref.window_attention((tok @ w.T + b)[:, perm], b[perm], table, B, X, Y, Z, C, heads, shift, head_major=True)
    torch.testing.assert_close(hm, got, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("B,X,Y,Z,shift", [(1, 11, 9, 2, True), (2, 8, 14, 1, False), (3, 4, 4, 1, True)])
def test_pieces_compose_to_port_swin_block(B, X, Y, Z, shift):
    """LayerNorm1 -> qkv_attention -> swin_tail (projection, residual, LN2, FFN, residual) = port.swin_block"""
    C, heads = 128, 4
    g = torch.Generator().manual_seed(ref.case_seed(B, X, Y, Z, 1))
    r = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)  # noqa: E731
    sd = {"norm1.weight": 1 + 0.1 * r(C), "norm1.bias": 0.1 * r(C), "norm2.weight": 1 + 0.1 * r(C),
          "norm2.bias": 0.1 * r(C), "attn.w_msa.qkv.weight": r(3 * C, C) * C ** -0.5, "attn.w_msa.qkv.bias": 0.3 * r(3 * C),
          "attn.w_msa.proj.weight": r(C, C) * C ** -0.5, "attn.w_msa.proj.bias": 0.1 * r(C),
          "attn.w_msa.relative_position_bias_table": r(169, heads),
          "ffn.layers.0.0.weight": r(C, C) * C ** -0.5, "ffn.layers.0.0.bias": 0.1 * r(C),
          "ffn.layers.1.weight": r(C, C) * C ** -0.5, "ffn.layers.1.bias": 0.1 * r(C)}
    tok = r(B * X * Y * (Z + 1), C)
    img = _images(tok, B, X, Y, Z).view(-1, X, Y, C).permute(0, 3, 1, 2)
    want = _rows(port.swin_block(img, sd, "", heads, shift).permute(0, 2, 3, 1).reshape(-1, X * Y, C), B, X, Y, Z)
    tokn = F.layer_norm(tok, (C,), sd["norm1.weight"], sd["norm1.bias"], ref.EPS)
    a = "attn.w_msa."
    att = ref.qkv_attention(tokn, sd[a + "qkv.weight"], sd[a + "qkv.bias"], sd[a + "relative_position_bias_table"],
                            B, X, Y, Z, C, heads, shift)
    got = ref.swin_tail(att, tok, sd[a + "proj.weight"], sd[a + "proj.bias"], sd["norm2.weight"], sd["norm2.bias"],
                        sd["ffn.layers.0.0.weight"], sd["ffn.layers.0.0.bias"], sd["ffn.layers.1.weight"],
                        sd["ffn.layers.1.bias"])
    torch.testing.assert_close(got, want, rtol=1e-10, atol=1e-10)


def test_plants_are_what_the_builder_says():
    """the large-logit window: keys outside a row's region outscore those inside by ~97 (so -100 leaves them ~e^-3 of the
    weight); the one-hot window: one key takes all but ~e^-60 of every unmasked row"""
    B, X, Y, Z, shift = ref.MISTAKE_CASE
    C, heads = 128, 4
    qkv, b, table, plants = ref.qkv_case(B, X, Y, Z, C, shift, ref.case_seed(B, X, Y, Z))
    rows, reg = ref.windows(B, X, Y, Z, shift)
    qkv = qkv.double()
    for name in ("large", "onehot"):
        r, g = rows[plants[name]], reg[plants[name]]
        src = torch.where((r < 0)[:, None], b.double(), qkv[r.clamp_min(0)])
        q, k, _ = src.view(ref.WT, 3, heads, ref.HD).permute(1, 2, 0, 3)
        s = (q @ k.transpose(-1, -2) * ref.SCALE)[0]
        if name == "large":
            out_reg = g[:, None] != g[None, :]
            real = (r >= 0)[:, None] & (r >= 0)[None, :]
            gap = s[out_reg & real].min() - s[~out_reg & real].max()
            assert 90 < float(gap) and float(s[out_reg & real].max() - s[~out_reg & real].min()) < 105
        else:
            t0 = int((r >= 0).nonzero()[0])
            others = torch.ones(ref.WT, dtype=torch.bool)
            others[t0] = False
            assert float((s[:, t0] - s[:, others].max(1).values).min()) > 55


# ------------------------------------------------------------------------------------------------ sensitivity
def _bites(mutant, want, what):
    r = rel_err(mutant, want)
    assert r > BITE, f"{what}: the planted mistake moves the result by only {r:.2e} (needs > {BITE:.0e})"


ATTN_MISTAKES = ["region threshold off by one", "-inf mask", "pad keys zero", "bias table transposed", "roll reversed",
                 "scale after the bias", "BEV image of the next sample"]


@pytest.mark.parametrize("kernel", ["window_attention", "qkv_attention"])
@pytest.mark.parametrize("mistake", ATTN_MISTAKES + ["phantom window's rows as keys"])
def test_attention_inputs_tell_planted_mistakes_apart(kernel, mistake):
    """the GPU test's MISTAKE_CASE (B = 3: BEV images of three samples; X, Y = 4, 5 mod 7: pad tokens; shift on), and for
    the phantom window its ODD_SHAPE case"""
    C, heads = 128, 4
    B, X, Y, Z, shift = (*ref.ODD_SHAPE, True) if mistake.startswith("phantom") else ref.MISTAKE_CASE
    assert not mistake.startswith("phantom") or ref.n_windows(B, X, Y, Z) % 2 == 1
    seed = ref.case_seed(B, X, Y, Z)
    if kernel == "window_attention":
        qkv, b, table, _ = ref.qkv_case(B, X, Y, Z, C, shift, seed)
        run = lambda m: ref.window_attention(qkv.double(), b.double(), table.double(), B, X, Y, Z, C, heads,  # noqa
                                             shift, mistake=m)
    else:
        tok, w, b, table, _ = ref.token_case(B, X, Y, Z, shift, seed)
        run = lambda m: ref.qkv_attention(tok.double(), w.double(), b.double(), table.double(), B, X, Y, Z, C,  # noqa
                                          heads, shift, mistake=m)
    _bites(run(mistake), run(None), f"{kernel}: {mistake}")


def test_masked_keys_keep_their_minus_100_weight():
    """in the large-logit window, the keys outside each row's region keep ~e^-3 of the weight: -inf would remove it"""
    B, X, Y, Z, shift = ref.MISTAKE_CASE
    qkv, b, table, plants = ref.qkv_case(B, X, Y, Z, 128, shift, ref.case_seed(B, X, Y, Z))
    rows, _ = ref.windows(B, X, Y, Z, shift)
    r = rows[plants["large"]]
    r = r[r >= 0]
    args = (qkv.double(), b.double(), table.double(), B, X, Y, Z, 128, 4, shift)
    _bites(ref.window_attention(*args, mistake="-inf mask")[r], ref.window_attention(*args)[r], "-inf, that window")


def _tail_views(out, M):
    """what the GPU test compares: the regular rows as one tensor, each special row on its own"""
    special = ref.tail_rows(M)
    keep = torch.ones(M, dtype=torch.bool)
    keep[list(special)] = False
    return [out[keep]] + [out[i:i + 1] for i in special]


@pytest.mark.parametrize("mistake", ["LN2 eps 1e-6", "tanh GELU", "b2 dropped"])
def test_tail_inputs_tell_planted_mistakes_apart(mistake):
    M = ref.TAIL_MISTAKE_M
    args = [t.double() for t in ref.tail_case(M, ref.case_seed(M))]
    want = ref.swin_tail(*args)
    kw = {"LN2 eps 1e-6": dict(eps=1e-6), "tanh GELU": dict(gelu_kind="tanh"), "b2 dropped": dict(with_b2=False)}
    got = ref.swin_tail(*args, **kw[mistake])
    moved = max(rel_err(g, w) for g, w in zip(_tail_views(got, M), _tail_views(want, M)))
    assert moved > BITE, f"{mistake}: moves the compared rows by only {moved:.2e} (needs > {BITE:.0e})"


def test_tail_case_reaches_both_gelu_tails_and_a_low_variance_row():
    M = ref.TAIL_MISTAKE_M
    att, tok, wp, bp, lw, lb, w1, b1, w2, b2 = (t.double() for t in ref.tail_case(M, ref.case_seed(M)))
    pre = ref.ffn_preact(att, tok, wp, bp, lw, lb, w1, b1)
    assert float(pre.min()) < -12 and float(pre.max()) > 7
    low, const, big = ref.tail_rows(M)
    y1 = tok + att @ wp.T + bp
    assert 0.5e-4 < float(y1[low].var(correction=0)) < 2e-4
    assert float(y1[const].std()) < 1e-6
    assert float(pre[const].max()) < -1.5 and float(pre[const].min()) > -4.5
    assert float(y1[big].mean()) > 500 * float(y1[big].std())
