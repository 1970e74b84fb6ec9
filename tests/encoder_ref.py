"""fp64 restatement of the dual-path encoder block's glue kernels (csrc/encoder_ops.cu), one launch at a time, in plain
torch (any device).

The functions take what a kernel is given, in fp64 and in the library's layouts, and return what that launch computes:
  - token rows: voxel rows ((b*X + x)*Y + y)*Z + z, then the BEV rows B*X*Y*Z + (b*X + x)*Y + y behind them;
  - GroupNorm statistics: fp64 (sum, sumsq) per (sample, group), packed (B, groups, 2), as the conv epilogue writes them;
  - S32 outputs are compared after decoding with ops.unsplit_weight.
tests/test_gpu_encoder_glue.py compares the kernels with them; tests/test_cpu_encoder_reference.py checks that they
compose to oracle.port.dualpath_block and that the GPU test's inputs tell planted mistakes apart, so a GPU failure points
at a kernel, not at the reference.  The input builders are shared by both files: the CPU check runs on the GPU test's
own inputs."""
import torch
import torch.nn.functional as F

EPS = 1e-5         # GroupNorm and LayerNorm eps of the reference modules
GATE_F32 = 1e-5    # kernel vs fp64, fp32 outputs (tests/util.assert_close, both criteria)
GATE_S32 = 2e-5    # kernel vs fp64, decoded S32 outputs (the split alone is within 2^-17 of each value)


# ------------------------------------------------------------------------------------------------ the launches
def gn_stats(x, B, groups):
    """x (B*rows_per_batch, C) -> fp64 (sum, sumsq) per (sample, group): (B, groups, 2)"""
    rows, C = x.shape
    v = x.double().view(B, rows // B, groups, C // groups)
    return torch.stack([v.sum((1, 3)), (v * v).sum((1, 3))], -1)


def group_norm(x, stats, w, b, rows_per_batch, groups, eps=EPS):
    """GroupNorm of x (B*rows_per_batch, C) with the mean / variance of stats (biased variance, clamped at 0), affine"""
    rows, C = x.shape
    B, cpg = rows // rows_per_batch, C // groups
    count = rows_per_batch * cpg
    mean = stats[..., 0] / count
    var = (stats[..., 1] / count - mean * mean).clamp_min(0)
    rstd = (var + eps).rsqrt()
    m = mean.repeat_interleave(cpg, 1).view(B, 1, C)
    r = rstd.repeat_interleave(cpg, 1).view(B, 1, C)
    return ((x.view(B, rows_per_batch, C) - m) * r * w + b).view(rows, C)


def layernorm(x, w, b, eps=EPS):
    """occ_layernorm"""
    return F.layer_norm(x, (x.shape[-1],), w, b, eps)


def gn_relu_zmean_ln(y, stats, gn_w, gn_b, ln_w, ln_b, B, XY, Z, groups, eps=EPS):
    """occ_gn_relu_zmean_ln: y (B*XY*Z, C) raw conv output -> (tok, tokn), both (B*XY*(Z+1), C) in token order:
    tok = ReLU(GroupNorm(y)) and its mean over Z (the BEV rows), tokn = LayerNorm1 of tok"""
    C = y.shape[1]
    v = torch.relu(group_norm(y, stats, gn_w, gn_b, XY * Z, groups, eps))
    tok = torch.cat([v, v.view(B * XY, Z, C).mean(1)])
    return tok, layernorm(tok, ln_w, ln_b, eps)


def gn_apply(x, stats, w, b, rows_per_batch, groups, residual=None, relu=True, eps=EPS):
    """occ_gn_apply: the GroupNorm affine, then the optional ReLU, then the optional residual"""
    o = group_norm(x, stats, w, b, rows_per_batch, groups, eps)
    if relu:
        o = torch.relu(o)
    return o if residual is None else o + residual


def pool_means(x, B):
    """per-sample column means of x (B*rows_per_batch, ch) -> (B, ch)"""
    return x.view(B, -1, x.shape[1]).mean(1)


def aspp_gap_values(means, wconv, gw, gb, groups, eps=EPS, correction=0):
    """the ASPP pool branch of per-sample means (B, ch): 1x1 conv wconv (ch, ch) -> GroupNorm over the 1x1 map (biased
    variance: correction 0, as torch's group_norm) -> ReLU -> (B, ch)"""
    B, ch = means.shape
    c = (means @ wconv.t()).view(B, groups, ch // groups)
    m = c.mean(-1, keepdim=True)
    var = c.var(-1, correction=correction, keepdim=True)
    return torch.relu(((c - m) * (var + eps).rsqrt()).view(B, ch) * gw + gb)


def aspp_gap_branch(x, wconv, gw, gb, B, groups, eps=EPS):
    """occ_aspp_gap_branch: per-sample mean -> 1x1 conv -> GroupNorm over a 1x1 map -> ReLU -> broadcast to every row of
    the sample: (B*rows_per_batch, ch), the values of the concat buffer's column slice"""
    v = aspp_gap_values(pool_means(x, B), wconv, gw, gb, groups, eps)
    return v.repeat_interleave(x.shape[0] // B, 0)


def depthnet_gap_branch(x, w, b, B):
    """occ_depthnet_gap_branch: per-image mean -> fc w (ch, ch) + b -> ReLU -> broadcast: (B*rows_per_batch, ch)"""
    v = torch.relu(pool_means(x, B) @ w.t() + b)
    return v.repeat_interleave(x.shape[0] // B, 0)


def dualpath_fuse(x, bev, cw, cbias, identity, B, XY, Z, id_stats=None, id_w=None, id_b=None, groups=0, eps=EPS):
    """occ_dualpath_fuse: x, identity (B*XY*Z, C) voxel rows, bev (B*XY, C) one row per column ->
    x + sigmoid(<x, cw> + cbias) * bev[row // Z] + identity, the identity GroupNorm'd (no ReLU) when id_stats is given"""
    coeff = torch.sigmoid(x @ cw + cbias)
    col = torch.arange(x.shape[0], device=x.device) // Z
    idn = identity if id_stats is None else group_norm(identity, id_stats, id_w, id_b, XY * Z, groups, eps)
    return x + coeff[:, None] * bev[col] + idn


# ------------------------------------------------------------------------------------------------ inputs
def case_seed(*case):
    """a fixed seed per test case (the same on CPU and GPU)"""
    s = 17
    for v in case:
        s = (s * 1000003 + int(v)) % (2 ** 31)
    return s


def gn_input(B, rows_per_batch, C, groups, seed, low_var=True):
    """fp32 (B*rows_per_batch, C): every (sample, group) has its own offset in [-2, 2) and scale in [0.5, 2), so sample
    and group mix-ups are visible; with low_var, group groups // 2 of the last sample has a variance near 1e-4, so an
    eps of 1e-6 instead of 1e-5 moves it by ~4%"""
    g = torch.Generator().manual_seed(seed)
    cpg = C // groups
    off = torch.rand(B, groups, generator=g, dtype=torch.float64) * 4 - 2
    scale = torch.rand(B, groups, generator=g, dtype=torch.float64) * 1.5 + 0.5
    if low_var:
        off[-1, groups // 2], scale[-1, groups // 2] = 0.02, 0.01
    x = torch.randn(B, rows_per_batch, groups, cpg, generator=g, dtype=torch.float64)
    return (x * scale[:, None, :, None] + off[:, None, :, None]).float().reshape(B * rows_per_batch, C)


def affine(C, seed):
    """(weight, bias) fp32 of a GroupNorm / LayerNorm"""
    g = torch.Generator().manual_seed(seed)
    return 1 + 0.1 * torch.randn(C, generator=g), 0.1 * torch.randn(C, generator=g)


def gn_case(B, rows_per_batch, C, groups):
    """fp32 (x, weight, bias) of a GroupNorm case: gn_input and affine with the case's own seeds"""
    return (gn_input(B, rows_per_batch, C, groups, case_seed(B, rows_per_batch, C, groups)),
            *affine(C, case_seed(C, groups)))


def gap_case(B, rows_per_batch, ch, groups):
    """fp32 (x, wconv (ch, ch), gn weight, gn bias) of a pool-branch case"""
    g = torch.Generator().manual_seed(case_seed(ch, groups))
    return (gn_input(B, rows_per_batch, ch, groups, case_seed(B, rows_per_batch, ch, groups)),
            torch.randn(ch, ch, generator=g) * ch ** -0.5, *affine(ch, case_seed(ch)))


def fuse_case(B, XY, Z, C, groups=32):
    """fp32 (x, bev, cw, identity) of a fusion case; the identity has per-(sample, group) offsets (the GroupNorm'd kind)"""
    g = torch.Generator().manual_seed(case_seed(B, XY, Z, C))
    x = torch.randn(B * XY * Z, C, generator=g)
    bev = torch.randn(B * XY, C, generator=g)
    cw = torch.randn(C, generator=g) * C ** -0.5
    return x, bev, cw, gn_input(B, XY * Z, C, groups, case_seed(B, XY, Z, C, groups))


def ln_rows(rows):
    """special rows of ln_input: (variance near 1e-4, constant, offset 1e3 x its spread); none below 4 rows"""
    return (1, rows // 2, rows - 1) if rows >= 4 else ()


def ln_input(rows, C, seed):
    """fp32 (rows, C) LayerNorm input: per-row offset in [-1, 1) and scale in [0.5, 2); the ln_rows() rows hold a row with
    a variance near 1e-4, a constant row (0.375: its sums are exact in fp32) and a row offset by 1e3 x its spread"""
    g = torch.Generator().manual_seed(seed)
    off = torch.rand(rows, 1, generator=g, dtype=torch.float64) * 2 - 1
    scale = torch.rand(rows, 1, generator=g, dtype=torch.float64) * 1.5 + 0.5
    x = torch.randn(rows, C, generator=g, dtype=torch.float64)
    special = ln_rows(rows)
    if special:
        low, const, big = special
        off[low], scale[low] = 0.01, 0.01
        off[big], scale[big] = 1e3, 1.0
        x[const], off[const], scale[const] = 0.375, 0.0, 1.0
    return (x * scale + off).float()
