"""fp64 restatement of the Swin attention and block-tail kernels (csrc/window_attn.cu, csrc/swin_attn_fused.cu,
csrc/swin_mlp_fused.cu), one launch at a time, in plain torch (any device).

The functions take what a kernel is given, in fp64 and in the library's token-row layout -- voxel rows
((b*X + x)*Y + y)*Z + z, then the BEV rows B*X*Y*Z + (b*X + x)*Y + y -- and return what that launch computes.  The
window attention is an explicit per-window gather: ShiftWindowMSA's pad, roll(-3, -3), region slices (0, -7), (-7, -3),
(-3, None) and window partition (window_attention.py:168-242) as index arithmetic, so it shares no code with
oracle.port.  S32 operands are decoded (ops.unsplit_weight) before they get here, so a gate measures only a kernel's
arithmetic.

tests/test_gpu_swin_attention.py compares the kernels with these functions; tests/test_cpu_swin_reference.py checks that
they equal oracle.port and that the GPU test's inputs tell planted mistakes apart.  `mistake` arguments exist for that
check only."""
import math

import torch
import torch.nn.functional as F

from encoder_ref import case_seed  # noqa: F401  (re-exported: one seed rule for every kernel-level test)

WS, WT, HD = 7, 49, 32
SHIFT = 3
SCALE = HD ** -0.5
MASK = -100.0          # additive shift mask of the reference (not -inf)
EPS = 1e-5             # LayerNorm eps of the reference modules
BIAS_FLOATS = 2404     # 49 * 49 bias values per head, padded to a 16-byte multiple
GATE = 5e-5            # kernel vs fp64 (tests/util.assert_close, both criteria): the GEMM / conv / neck-tail gate
BF16_GATE = 3e-2       # single-pass bf16 mode (ops.precision("bf16")) vs fp64
TAIL_C = 128
PLANT_CH = 6           # token channels 0..5 carry the planted windows of token_case


# ------------------------------------------------------------------------------------------------ window geometry
def grid(X, Y):
    """-> (nWx, nWy, Xp, Yp): windows per axis and the padded extent"""
    nWx, nWy = -(-X // WS), -(-Y // WS)
    return nWx, nWy, nWx * WS, nWy * WS


def n_windows(B, X, Y, Z):
    nWx, nWy, _, _ = grid(X, Y)
    return B * (Z + 1) * nWx * nWy


def _region(n_pad, shift, inner):
    """shift-mask region along one axis of the rolled, padded image: slices (0, -7) -> 0, (-7, -inner) -> 1, (-inner,
    None) -> 2 (inner = 3 in the reference)"""
    s = torch.arange(n_pad)
    if not shift:
        return torch.zeros(n_pad, dtype=torch.long)
    return torch.where(s < n_pad - WS, 0, torch.where(s < n_pad - inner, 1, 2))


def windows(B, X, Y, Z, shift, mistake=None):
    """-> (rows, region), each (B*(Z+1), nWx, nWy, 49) int64: the token row behind position t = 7i + j of window (wx, wy)
    of image img (-1 for a pad token) and its shift-mask region.  Images: (b, z) voxel slices b*Z + z, then the B BEV
    images.  The rolled image holds at (xs, ys) the padded image's (xs + 3, ys + 3) mod (Xp, Yp)."""
    nWx, nWy, Xp, Yp = grid(X, Y)
    s = (-SHIFT if mistake == "roll reversed" else SHIFT) if shift else 0
    inner = SHIFT + 1 if mistake == "region threshold off by one" else SHIFT
    x = ((torch.arange(Xp) + s) % Xp).view(nWx, 1, WS, 1).expand(nWx, nWy, WS, WS)
    y = ((torch.arange(Yp) + s) % Yp).view(1, nWy, 1, WS).expand(nWx, nWy, WS, WS)
    reg = (_region(Xp, shift, inner).view(nWx, 1, WS, 1) * 3 + _region(Yp, shift, inner).view(1, nWy, 1, WS))
    reg = reg.expand(nWx, nWy, WS, WS).reshape(1, nWx, nWy, WT)
    pad = ((x >= X) | (y >= Y)).reshape(1, nWx, nWy, WT)
    x, y = x.reshape(1, nWx, nWy, WT), y.reshape(1, nWx, nWy, WT)
    img = torch.arange(B * (Z + 1)).view(-1, 1, 1, 1)
    vox = img < B * Z
    bev_b = img - B * Z
    if mistake == "BEV image of the next sample":
        bev_b = (bev_b + 1) % B
    rows = torch.where(vox, (((img // Z) * X + x) * Y + y) * Z + img % Z, B * X * Y * Z + (bev_b * X + x) * Y + y)
    rows = rows.masked_fill(pad, -1)
    return rows, reg.expand(rows.shape)


def rel_index():
    """(49, 49) index into the (13*13, heads) relative-position bias table: 13 (i_a - i_b + 6) + (j_a - j_b + 6)"""
    i, j = torch.arange(WT) // WS, torch.arange(WT) % WS
    return 13 * (i[:, None] - i[None, :] + WS - 1) + (j[:, None] - j[None, :] + WS - 1)


def dense_bias(table):
    """(169, heads) table -> (heads, 49 queries, 49 keys)"""
    return table[rel_index().to(table.device)].permute(2, 0, 1)


def bias_pad(table):
    """the kernels' bias operand: (heads, 2404) fp32, 49 x 49 per head, zero padded"""
    d = dense_bias(table.float()).reshape(table.shape[1], WT * WT)
    return F.pad(d, (0, BIAS_FLOATS - WT * WT)).contiguous()


def head_major_perm(C, heads):
    """row permutation of the qkv weight / bias: head-major row h*96 + which*32 + d <- reference row which*C + h*32 + d"""
    return torch.arange(3 * C).view(3, heads, HD).permute(1, 0, 2).reshape(-1)


# ------------------------------------------------------------------------------------------------ the launches
def window_attention(qkv, qkv_bias, table, B, X, Y, Z, C, heads, shift, head_major=False, mistake=None, chunk=4096,
                     with_abs=False):
    """occ_window_attention: qkv (rows, 3C) token rows, qkv_bias (3C,), table (169, heads) -> (rows, C).
    Columns [q | k | v][head][32] (reference order) or [head][q | k | v][32] (head_major).  Pad tokens take qkv = bias.
    with_abs: -> (out, P |V|), the second the scale of the P V error (pv_error)."""
    dev = qkv.device
    if head_major:
        perm = head_major_perm(C, heads).to(dev)
        ref_qkv, ref_b = torch.empty_like(qkv), torch.empty_like(qkv_bias)
        ref_qkv[:, perm], ref_b[perm] = qkv, qkv_bias
        qkv, qkv_bias = ref_qkv, ref_b
    rows, reg = windows(B, X, Y, Z, shift, mistake)
    # a BEV image gathered from the next sample's rows, but written to its own
    dst = windows(B, X, Y, Z, shift)[0] if mistake == "BEV image of the next sample" else rows
    rows, reg, dst = rows.reshape(-1, WT).to(dev), reg.reshape(-1, WT).to(dev), dst.reshape(-1, WT).to(dev)
    nwin = rows.shape[0]
    bias = dense_bias(table)
    if mistake == "bias table transposed":
        bias = bias.transpose(1, 2)
    pad_src = torch.zeros_like(qkv_bias) if mistake == "pad keys zero" else qkv_bias
    out = torch.zeros(qkv.shape[0], C, dtype=qkv.dtype, device=dev)
    out_abs = torch.zeros_like(out) if with_abs else None
    for w0 in range(0, nwin, chunk):
        r, g = rows[w0:w0 + chunk], reg[w0:w0 + chunk]
        n = r.shape[0]
        src = torch.where((r < 0)[..., None], pad_src, qkv[r.clamp_min(0)])
        q, k, v = src.view(n, WT, 3, heads, HD).permute(2, 0, 3, 1, 4)
        if mistake == "scale after the bias":
            s = (q @ k.transpose(-1, -2) + bias) * SCALE
        else:
            s = (q * SCALE) @ k.transpose(-1, -2) + bias
        diff = (g[:, :, None] != g[:, None, :])[:, None]
        s = s.masked_fill(diff, -math.inf) if mistake == "-inf mask" else s + diff * MASK
        if mistake == "phantom window's rows as keys" and nwin % 2 and w0 + n == nwin:
            # the odd last window also attends to its partner in the pair: 49 zero rows (score 0, v = 0)
            s = torch.cat([s, torch.zeros_like(s).masked_fill(torch.arange(n, device=dev)[:, None, None, None] < n - 1,
                                                              -math.inf)], -1)
            v = torch.cat([v, torch.zeros_like(v)], -2)
        p = s.softmax(-1)
        o = (p @ v).transpose(1, 2).reshape(n, WT, C)
        d = dst[w0:w0 + chunk]
        ok = d >= 0
        out[d[ok]] = o[ok]
        if with_abs:
            out_abs[d[ok]] = (p @ v.abs()).transpose(1, 2).reshape(n, WT, C)[ok]
    return (out, out_abs) if with_abs else out


def s32(t):
    """the values an fp32 tensor keeps in the S32 split format: fp32, then bf16 hi + bf16 lo of the remainder (fp64)"""
    f = t.float()
    hi = f.bfloat16().float()
    return (hi.double() + (f - hi).bfloat16().double())


def qkv_attention(tokens, w_qkv, b_qkv, table, B, X, Y, Z, C, heads, shift, mistake=None, split_qkv=False,
                  with_abs=False):
    """occ_swin_qkv_attention: the projection tokens W^T + b (reference-order rows), then window_attention.  Pad tokens
    are zero rows of the window layout, so their q / k / v are the bias.  split_qkv: q / k / v as the attention core
    consumes them -- the kernel rounds the projection to fp32 and splits it to bf16 hi + lo (the S32 hand-off of the
    two-kernel path), so only lo * lo and the accumulations remain for the gate to measure."""
    qkv, b = tokens @ w_qkv.T + b_qkv, b_qkv
    if split_qkv:
        qkv, b = s32(qkv), s32(b)
    return window_attention(qkv, b, table, B, X, Y, Z, C, heads, shift, mistake=mistake, with_abs=with_abs)


def gelu(x, kind="erf"):
    return F.gelu(x, approximate="tanh" if kind == "tanh" else "none")


def swin_tail(att, tok, wp, bp, ln_w, ln_b, w1, b1, w2, b2, eps=EPS, gelu_kind="erf", with_b2=True):
    """occ_swin_proj_ffn: y1 = tok + att Wp^T + bp;  y1 + W2 GELU(W1 LN2(y1) + b1) + b2"""
    y1 = tok + att @ wp.T + bp
    h = gelu(F.layer_norm(y1, (y1.shape[1],), ln_w, ln_b, eps) @ w1.T + b1, gelu_kind)
    return y1 + h @ w2.T + (b2 if with_b2 else 0)


def ffn_preact(att, tok, wp, bp, ln_w, ln_b, w1, b1):
    """the GELU inputs of swin_tail"""
    y1 = tok + att @ wp.T + bp
    return F.layer_norm(y1, (y1.shape[1],), ln_w, ln_b, EPS) @ w1.T + b1


# ------------------------------------------------------------------------------------------------ error model
def qk_split_bound(qkv, qkv_bias, B, X, Y, Z, C, heads, shift, window):
    """largest score error of the hi / lo products in one window: the three passes hi*hi + lo*hi + hi*lo drop lo * lo,
    and |lo| <= 2^-9 |.|, so |ds| <= 2^-18 * scale * sum_d |q_d| |k_d|.  Zero for bf16-exact q, k (lo = 0), as in
    qkv_case's planted windows; not for the q, k the fused kernel computes.  -> that bound (qkv as the core consumes it,
    reference-order columns)"""
    rows, _ = windows(B, X, Y, Z, shift)
    r = rows[window].to(qkv.device)
    src = torch.where((r < 0)[:, None], qkv_bias, qkv[r.clamp_min(0)])
    q, k, _ = src.view(WT, 3, heads, HD).permute(1, 2, 0, 3).abs()
    return float(2.0 ** -18 * SCALE * (q @ k.transpose(-1, -2)).max())


def pv_error(p_abs_v):
    """bound on what the split P V product of both attention kernels adds to an output element, from P |V| (with_abs):
    P is kept as bf16 hi + lo (<= 2^-18 |p| lost), the three passes drop P_lo V_lo (<= 2^-18 |p||v|), and ex2.approx,
    the fp32 accumulation and the final S32 split of the output add a few 2^-22 more: <= 2^-16 sum_j p_j |v_j|.  It
    scales with the values averaged, not with the output, so where the output is a small average of large values this
    exceeds the allclose criterion's GATE * (rms + |out|)."""
    return 2.0 ** -16 * p_abs_v


# ------------------------------------------------------------------------------------------------ inputs
def plant_windows(B, X, Y, Z, shift):
    """(img, wx, wy) of each planted window (a window gets at most one plant; one that would collide is left out):
    large  -- image 0, the last window row: under shift it straddles the regions rx = 1 / 2
    onehot -- image 1, window (0, 0)
    uniform -- the last image (a BEV image), the last window
    pad    -- the second-to-last image, the window with the most pad tokens (none without pad tokens)"""
    nWx, nWy, _, _ = grid(X, Y)
    nimg = B * (Z + 1)
    rows, _ = windows(B, X, Y, Z, shift)
    npad = (rows[0] < 0).sum(-1)
    want = {"large": (0, nWx - 1, 0), "onehot": (1, 0, 0), "uniform": (nimg - 1, nWx - 1, nWy - 1)}
    if int(npad.max()) > 0:
        i = int(npad.flatten().argmax())
        want["pad"] = (max(nimg - 2, 0), i // nWy, i % nWy)
    out = {}
    for name, w in want.items():
        if w not in out.values():
            out[name] = w
    return out


def token_case(B, X, Y, Z, shift, seed):
    """C = 128 inputs of the fused kernel: (tokens (rows, 128), w_qkv (384, 128) and b_qkv (384,) in reference-order
    rows, table (169, 4), plants), fp32.  Random tokens and weights, except token channels 0..5, which are zero outside
    the planted windows (channel 5: 1 in every real token), and these qkv rows of every head h, which read one channel:
      q0 = 4 x0, q1 = 4 x1, k0 = 4 x1, k1 = 4 x0   large : rows of token 0's region x0 = a, the others x1 = a; a^2 16 =
                                                            549, so keys outside a row's region outscore those inside by
                                                            549 * 32^-0.5 = 97 (-100 leaves them ~e^-3 of the weight,
                                                            -inf none)
      q2 = 4 x2, k2 = 4 x3                         onehot: every row x2 = a', the first real token x3 = a': it outscores
                                                            the window's other keys by 60
      q4 = 4 x4, k4 = 4 (bias) - 4 x5              pad   : rows x4 = 2: pad keys (k4 = 4, real keys k4 = 0) score 5.7 up
    uniform: every token of the window is zero, so q = k = v = bias."""
    C, heads = TAIL_C, TAIL_C // HD
    g = torch.Generator().manual_seed(seed)
    rows = B * X * Y * (Z + 1)
    tok = torch.randn(rows, C, generator=g, dtype=torch.float64)
    tok[:, :PLANT_CH] = 0
    tok[:, 5] = 1
    w = torch.randn(3 * C, C, generator=g, dtype=torch.float64) * C ** -0.5
    w[:, :PLANT_CH] = 0
    b = 0.3 * torch.randn(3 * C, generator=g, dtype=torch.float64)
    table = torch.randn(169, heads, generator=g, dtype=torch.float64)
    gam = 4.0
    for h in range(heads):
        q, k = h * HD, C + h * HD
        for row, col in ((q, 0), (q + 1, 1), (k, 1), (k + 1, 0), (q + 2, 2), (k + 2, 3), (q + 4, 4), (k + 4, 5)):
            w[row] = 0
            w[row, col] = -gam if (row, col) == (k + 4, 5) else gam
            b[row] = 0
        b[k + 4] = gam
    a_large, a_one = math.sqrt(549.0) / gam, math.sqrt(340.0) / gam
    wrows, wreg = windows(B, X, Y, Z, shift)
    plants = plant_windows(B, X, Y, Z, shift)
    for name, (img, wx, wy) in plants.items():
        r, reg = wrows[img, wx, wy], wreg[img, wx, wy]
        real = r >= 0
        rr = r[real]
        if name == "large":
            same = (reg == reg[0])[real]
            tok[rr[same], 0] = a_large
            tok[rr[~same], 1] = a_large
        elif name == "onehot":
            tok[rr, 2] = a_one
            tok[rr[0], 3] = a_one
        elif name == "pad":
            tok[rr, 4] = 2.0
        elif name == "uniform":
            tok[rr] = 0
    return tok.float(), w.float(), b.float(), table.float(), plants


def qkv_case(B, X, Y, Z, C, shift, seed):
    """inputs of occ_window_attention: (qkv (rows, 3C) fp32 token rows, qkv_bias (3C,), table (169, heads), plants).
    C = 128: the projection of token_case, with the rows of the planted windows rounded to bf16, so that their
    products are exact and the large-logit window has no operand-split error; other C: random qkv (unit variance), bias
    0.3 randn."""
    if C == TAIL_C:
        tok, w, b, table, plants = token_case(B, X, Y, Z, shift, seed)
        qkv = (tok.double() @ w.double().T + b.double()).float()
        wrows, _ = windows(B, X, Y, Z, shift)
        for img, wx, wy in plants.values():
            r = wrows[img, wx, wy]
            r = r[r >= 0]
            qkv[r] = qkv[r].bfloat16().float()
        return qkv, b, table, plants
    g = torch.Generator().manual_seed(seed)
    rows = B * X * Y * (Z + 1)
    return (torch.randn(rows, 3 * C, generator=g), 0.3 * torch.randn(3 * C, generator=g),
            torch.randn(169, C // HD, generator=g), {})


def tail_rows(M):
    """special rows of tail_case: (LN2 variance near 1e-4, constant, offset 1e3 x its spread); none below 4 rows"""
    return (1, M // 2, M - 1) if M >= 4 else ()


def tail_case(M, seed):
    """fp32 (att, tok, wp, bp, ln_w, ln_b, w1, b1, w2, b2) of occ_swin_proj_ffn, C = 128.  W1 has gain 3 and b1 is
    centred at -3, so the GELU inputs span about -15 .. +9 (both tails of smf_gelu).  The tail_rows() rows: y1 with a
    variance near 1e-4 (LN2's eps of 1e-5 vs 1e-6 moves its output by ~4 %), a constant y1 (LN2 output = ln_b: every GELU
    input within about -4 .. -2, where the erf and tanh forms differ by 10 %), and y1 offset by 1e3 x its spread; att is zero in the
    first two, so the kernel's y1 = tok + bp carries one fp32 rounding and no GEMM error."""
    C = TAIL_C
    g = torch.Generator().manual_seed(seed)
    att = torch.randn(M, C, generator=g, dtype=torch.float64)
    tok = torch.randn(M, C, generator=g, dtype=torch.float64)
    wp = torch.randn(C, C, generator=g, dtype=torch.float64) * C ** -0.5
    w1 = 3 * torch.randn(C, C, generator=g, dtype=torch.float64) * C ** -0.5
    w2 = torch.randn(C, C, generator=g, dtype=torch.float64) * C ** -0.5
    bp, b2 = (0.1 * torch.randn(C, generator=g, dtype=torch.float64) for _ in range(2))
    b1 = -3 + 0.1 * torch.randn(C, generator=g, dtype=torch.float64)
    lw, lb = 1 + 0.1 * torch.randn(C, generator=g, dtype=torch.float64), 0.1 * torch.randn(C, generator=g,
                                                                                             dtype=torch.float64)
    special = tail_rows(M)
    bp32 = bp.float().double()
    if special:
        low, const, big = special
        att[low] = att[const] = 0
        tok[low] = (0.3 + 0.01 * torch.randn(C, generator=g, dtype=torch.float64)) - bp32
        tok[const] = 0.375 - bp32
        tok[big] = 1e3 + tok[big]
    return tuple(t.float() for t in (att, tok, wp, bp, lw, lb, w1, b1, w2, b2))


# ------------------------------------------------------------------------------------------------ the GPU test's cases
# (B, X, Y, Z): X mod 7 and Y mod 7 each take every residue 0..6 (the nuScenes 200-grid and its stage-3 25, and KITTI's
# stage-2 32, are 4 mod 7), X, Y < 7, B = 1, 2, 3; run with the shift on and off
RESIDUE_SHAPES = [(1, 7, 11, 1), (2, 8, 13, 1), (3, 9, 7, 1), (1, 10, 9, 2), (3, 11, 12, 1), (2, 12, 8, 2),
                  (1, 13, 10, 1), (3, 3, 5, 2), (2, 6, 2, 1), (1, 4, 4, 3)]
ODD_SHAPE = (1, 15, 15, 2)        # B = 1, Z even, nWx and nWy odd: 27 windows, the last pair holds a phantom window
MISTAKE_CASE = (3, 11, 12, 1, True)
TAIL_MISTAKE_M = 1000
