"""fp64 restatement of the pixel decoder's (MSDeformAttnPixelDecoder3D) non-GEMM kernels (csrc/neck_ops.cu and
occ_gn_stats), one launch at a time, in plain torch (any device).

The functions take what a kernel is given, in fp64 and in the library's layouts, and return what that launch computes:
  - token rows are level-major: row(l, b, x, y, z) = B*start_l + b*n_l + (x*Y_l + y)*Z_l + z, levels coarse -> fine;
  - GroupNorm statistics: fp64 (sum, sumsq) per (sample, group), packed (B, groups, 2);
  - S32 outputs are compared after decoding with ops.unsplit_weight.
tests/test_gpu_neck_ops.py compares the kernels with them; tests/test_cpu_neck_reference.py checks that they compose to
oracle.port's encoder layer and FPN step and that the GPU test's inputs tell planted mistakes apart.  The input builders
are shared by both files: the CPU check runs on the GPU test's own inputs.

`mistake` arguments plant one named error in a reference launch; only the CPU sensitivity test passes them."""
import math

import torch

from encoder_ref import EPS, GATE_F32, GATE_S32, affine, case_seed, group_norm, ln_input, ln_rows  # noqa: F401


# ------------------------------------------------------------------------------------------------ layout
def level_starts(grids):
    """first token of every level inside one sample's Nq tokens"""
    ns = [x * y * z for x, y, z in grids]
    return [sum(ns[:i]) for i in range(len(ns))], ns


def pos_index(grids, B, device=None, mistake=None):
    """the pos row of every level-major token row: start_l + local, independent of the sample.
    mistake "sample_major": the row read as if the tokens were stored sample by sample (row % Nq)"""
    starts, ns = level_starts(grids)
    if mistake == "sample_major":
        return torch.arange(B * sum(ns), device=device) % sum(ns)
    return torch.cat([torch.arange(n, device=device).repeat(B) + s for s, n in zip(starts, ns)])


def row_coords(grids, B, device=None):
    """per level-major row: (level, sample, x, y, z) as int64 tensors"""
    out = []
    for lvl, (X, Y, Z) in enumerate(grids):
        i = torch.arange(B * X * Y * Z, device=device)
        b, loc = i // (X * Y * Z), i % (X * Y * Z)
        out.append(torch.stack([torch.full_like(i, lvl), b, loc // (Y * Z), (loc // Z) % Y, loc % Z], 1))
    return torch.cat(out).unbind(1)


# ------------------------------------------------------------------------------------------------ the launches
def gn_stats(x, B, groups, mistake=None):
    """occ_gn_stats: x (B*rows_per_sample, C) -> fp64 (sum, sumsq) per (sample, group): (B, groups, 2).
    mistake "next_sample": the rows of sample b + 1 are counted in sample b as well"""
    rows, C = x.shape
    v = x.double().view(B, rows // B, groups, C // groups)
    st = torch.stack([v.sum((1, 3)), (v * v).sum((1, 3))], -1)
    if mistake == "next_sample":
        st = st.clone()
        st[:-1] += st[1:].clone()
    return st


def token_prep(x, grids, B, ln=None, pos=None, eps=EPS, mistake=None):
    """occ_neck_token_prep: [LayerNorm (biased variance, eps)] of every row -> (y, y + pos[start_l + local] or None).
    mistake "pos_sample_major": pos row of a sample-major layout; "pos_before_ln": the LayerNorm of x + pos"""
    idx = pos_index(grids, B, x.device, "sample_major" if mistake == "pos_sample_major" else None)
    y = x + pos[idx] if mistake == "pos_before_ln" else x
    if ln is not None:
        m = y.mean(-1, keepdim=True)
        var = ((y - m) ** 2).mean(-1, keepdim=True)
        y = (y - m) * (var + eps).rsqrt() * ln[0] + ln[1]
    if pos is None:
        return y, None
    return y, (y if mistake == "pos_before_ln" else y + pos[idx])


def ref_points(grids, strides, dtype=torch.float64, device=None):
    """reference point of every query token of one sample, (Nq, 3) columns (z, y, x): its voxel centre normalised in its
    own level, computed as the kernel does, ((i + 0.5) * stride) / (n * stride)"""
    out = []
    for (X, Y, Z), s in zip(grids, strides):
        ax = [((torch.arange(n, dtype=dtype, device=device) + 0.5) * s) / (n * s) for n in (X, Y, Z)]
        gx, gy, gz = torch.meshgrid(*ax, indexing="ij")
        out.append(torch.stack([gz.reshape(-1), gy.reshape(-1), gx.reshape(-1)], -1))
    return torch.cat(out)


MSDA_MISTAKES = ("align_corners", "offset_xyz", "ref_value_level", "border", "softmax_per_level", "sample0", "swap_t")


def ms_deform_attn(value, ow, grids, strides, B, E, H, P=4, head_ld=None, chunk=2048, mistake=None, coords="fp64"):
    """occ_ms_deform_attn: value (rows, >= H*head_ld) with head h in columns [h*head_ld, h*head_ld + E/H); ow (rows,
    H*L*P*4) = [offsets (h, l, p, (z, y, x)) | logits (h, l, p)]; -> (rows, E) = sum over the L*P points of a head of
    softmax(logits) * trilinear(value of level l)(loc), loc = ref + offset / (Z_l, Y_l, X_l), un-normalised as grid_sample
    with align_corners=False (f = loc * n - 0.5), zeros outside.  An explicit 8-corner gather (no F.grid_sample), in
    query chunks of `chunk` rows.  mistake: one of MSDA_MISTAKES (test_cpu_neck_reference.py).
    coords "fp32": the sampling coordinate f is computed with the kernel's fp32 operations, as the fp32 model computes
    its sampling locations (everything after f stays fp64).  On a 100-voxel axis an fp32 location is only known to
    ~6e-6 voxel, which moves an output by up to ~1e-5 of the value spread: more than the S32 gate allows next to a small
    output, and a property of the fp32 operation, not of the kernel."""
    L = len(grids)
    hd = E // H
    head_ld = hd if head_ld is None else head_ld
    dev, rows = value.device, value.shape[0]
    cols = (torch.arange(H, device=dev)[:, None] * head_ld + torch.arange(hd, device=dev)).reshape(-1)
    V = value[:, cols].double().reshape(rows, H, hd)
    starts, ns = level_starts(grids)
    lvl, b, x, y, z = row_coords(grids, B, dev)
    dims = torch.tensor([[Z, Y, X] for X, Y, Z in grids], dtype=torch.float64, device=dev)  # (L, 3) as (z, y, x)
    st = torch.tensor([float(s) for s in strides], dtype=torch.float64, device=dev)
    out = torch.empty(rows, H, hd, dtype=torch.float64, device=dev)
    hidx = torch.arange(H, device=dev)[None, :, None]
    for r0 in range(0, rows, chunk):
        sl = slice(r0, min(rows, r0 + chunk))
        n = sl.stop - sl.start
        o = ow[sl].double()
        off = o[:, :H * L * P * 3].reshape(n, H, L, P, 3)
        logit = o[:, H * L * P * 3:].reshape(n, H, L, P)
        if mistake == "softmax_per_level":
            w = logit.softmax(-1)
        else:
            w = logit.reshape(n, H, L * P).softmax(-1).reshape(n, H, L, P)
        ql, qb = lvl[sl], b[sl]
        qi = torch.stack([z[sl], y[sl], x[sl]], 1).double()  # (n, 3) voxel index in the query level, (z, y, x)
        s = st[ql][:, None]
        ref = ((qi + 0.5) * s) / (dims[ql] * s)
        if coords == "fp32":
            ref32 = ((qi.float() + 0.5) * s.float()) / (dims[ql].float() * s.float())
        if mistake == "sample0":
            qb = torch.zeros_like(qb)
        acc = torch.zeros(n, H, hd, dtype=torch.float64, device=dev)
        for l in range(L):
            Zl, Yl, Xl = grids[l][2], grids[l][1], grids[l][0]
            d = dims[l]
            r = ((qi + 0.5) * s) / (d * s) if mistake == "ref_value_level" else ref
            norm = d.flip(0) if mistake == "offset_xyz" else d
            if coords == "fp32":  # the kernel's float ops: ((2 loc - 1) + 1) * n - 1 as one fma, then * 0.5
                loc = ref32[:, None, None, :] + off[:, :, l].float() / d.float()
                f = (((2 * loc - 1) + 1).double() * d - 1).float().double() * 0.5
            else:
                loc = r[:, None, None, :] + off[:, :, l] / norm  # (n, H, P, 3)
                f = loc * (d - 1) if mistake == "align_corners" else loc * d - 0.5
            if mistake == "border":
                f = torch.minimum(f.clamp_min(0), d - 1)
            f0 = torch.floor(f)
            t = f - f0
            if mistake == "swap_t":
                t = torch.cat([1 - t[..., :1], t[..., 1:]], -1)
            i0 = torch.minimum(f0.clamp_min(-2), d).long()  # beyond the volume either way: every corner is dropped
            base = (B * starts[l] + qb * ns[l])[:, None, None]
            wl = w[:, :, l]
            for k in range(8):
                dz, dy, dx = k & 1, (k >> 1) & 1, k >> 2
                zz, yy, xx = i0[..., 0] + dz, i0[..., 1] + dy, i0[..., 2] + dx
                ok = (zz >= 0) & (zz < Zl) & (yy >= 0) & (yy < Yl) & (xx >= 0) & (xx < Xl)
                cw = ((t[..., 0] if dz else 1 - t[..., 0]) * (t[..., 1] if dy else 1 - t[..., 1]) *
                      (t[..., 2] if dx else 1 - t[..., 2]))
                row = torch.where(ok, base + (xx * Yl + yy) * Zl + zz, 0)
                cw = torch.where(ok, cw * wl, 0.0)
                acc += (cw[..., None] * V[row, hidx]).sum(2)
        out[sl] = acc
    return out.reshape(rows, E)


def upsample_axis(n_out, n_in, device=None, mistake=None):
    """F.interpolate's align_corners=False source index on one axis: src = (d + 0.5) * (n_in / n_out) - 0.5 clamped at 0,
    i0 = floor, i1 = i0 + 1 clamped to the last element -> (i0, i1, t).
    mistake "align_corners": src = d * (n_in - 1) / (n_out - 1); "nearest": floor(d * n_in / n_out), t = 0;
    "no_clamp": src not clamped at 0 (truncated to i0 = 0, so t < 0 extrapolates)"""
    d = torch.arange(n_out, dtype=torch.float64, device=device)
    if mistake == "nearest":
        i0 = torch.floor(d * (n_in / n_out)).long().clamp_max(n_in - 1)
        return i0, i0, torch.zeros_like(d)
    if mistake == "align_corners":
        src = d * ((n_in - 1) / (n_out - 1)) if n_out > 1 else torch.zeros_like(d)
    else:
        src = (d + 0.5) * (n_in / n_out) - 0.5
        if mistake != "no_clamp":
            src = src.clamp_min(0)
    i0 = torch.trunc(src).long().clamp_max(n_in - 1)
    i1 = (i0 + 1).clamp_max(n_in - 1)
    return i0, i1, src - i0


GN_UP_MISTAKES = ("align_corners", "nearest", "no_clamp")


def gn_upsample_add(cur, stats, gw, gb, groups, coarse, eps=EPS, mistake=None):
    """occ_gn_upsample_add: cur (B, X, Y, Z, C) raw lateral conv output, stats its (B, groups, 2) GroupNorm statistics,
    coarse (B, Xc, Yc, Zc, C) -> GroupNorm(cur) + trilinear upsample (align_corners=False) of coarse, (B, X, Y, Z, C).
    mistake: one of GN_UP_MISTAKES (upsample_axis)"""
    B, X, Y, Z, C = cur.shape
    _, Xc, Yc, Zc, _ = coarse.shape
    gn = group_norm(cur.reshape(-1, C), stats, gw, gb, X * Y * Z, groups, eps).view(B, X, Y, Z, C)
    (x0, x1, tx), (y0, y1, ty), (z0, z1, tz) = (upsample_axis(o, i, cur.device, mistake)
                                                for o, i in ((X, Xc), (Y, Yc), (Z, Zc)))
    up = torch.zeros_like(gn)
    for k in range(8):
        dz, dy, dx = k & 1, (k >> 1) & 1, k >> 2
        xi, yi, zi = (x1 if dx else x0), (y1 if dy else y0), (z1 if dz else z0)
        w = ((tx if dx else 1 - tx)[:, None, None] * (ty if dy else 1 - ty)[None, :, None] *
             (tz if dz else 1 - tz)[None, None, :])
        up += w[None, ..., None] * coarse[:, xi][:, :, yi][:, :, :, zi]
    return gn + up


# ------------------------------------------------------------------------------------------------ inputs
def gn_input(B, rows_per_sample, C, groups, seed):
    """fp32 (B*rows_per_sample, C): every (sample, group) has its own offset in [-2, 2) and scale in [0.5, 2), so sample
    and group mix-ups are visible.  gn_special() names two planted groups: group groups // 2 of the last sample has mean
    1 and std 1e-2 (variance 1e-4: eps 1e-6 instead of 1e-5 moves it by ~4%; mean / std = 100) and, with two or more
    groups, group 0 of the first sample has mean 30 and std 0.3 (mean / std = 100 at a larger magnitude)"""
    g = torch.Generator().manual_seed(seed)
    cpg = C // groups
    off = torch.rand(B, groups, generator=g, dtype=torch.float64) * 4 - 2
    scale = torch.rand(B, groups, generator=g, dtype=torch.float64) * 1.5 + 0.5
    for (b, gi), (m, s) in zip(gn_special(B, groups), ((1.0, 1e-2), (30.0, 0.3))):
        off[b, gi], scale[b, gi] = m, s
    x = torch.randn(B, rows_per_sample, groups, cpg, generator=g, dtype=torch.float64)
    return (x * scale[:, None, :, None] + off[:, None, :, None]).float().reshape(B * rows_per_sample, C)


def gn_special(B, groups):
    """(sample, group) of gn_input's planted groups: the small-variance group, then the offset group"""
    return [(B - 1, groups // 2)] + ([(0, 0)] if groups > 1 else [])


def token_input(grids, B, C, seed):
    """fp32 level-major rows (B*Nq, C) from ln_input (per-row offset and scale; a row with a variance near 1e-4, a
    constant row and a row offset by 1e3 x its spread at ln_rows(rows)) and pos (Nq, C)"""
    rows = B * sum(x * y * z for x, y, z in grids)
    g = torch.Generator().manual_seed(seed + 1)
    return ln_input(rows, C, seed), torch.randn(rows // B, C, generator=g)


# un-normalised per-axis targets of the planted sampling points (in voxels of the value level; n = its size)
_KINDS = ("centre", "face_lo", "face_hi", "out_lo", "out_hi", "far_lo", "far_hi", "huge_lo", "huge_hi")


def _target(kind, n, k):
    return {"centre": float(k % n), "face_lo": -0.5, "face_hi": n - 0.5, "out_lo": -0.75, "out_hi": n - 0.25,
            "far_lo": -1e4, "far_hi": n + 1e4}[kind]


def ow_input(grids, B, H, P=4, seed=0, planted=0.3):
    """fp32 (rows, H*L*P*4) sampling offsets and attention logits.  Offsets are N(0, 1.5) voxels, except that on every
    axis of every point a fraction `planted` is replaced by a planted target (_KINDS): a voxel centre, exactly a face
    (-0.5, n - 0.5), 0.25 voxel outside a face, 1e4 voxels out, or an offset of +-1e30 (the kernel's int clamp); levels
    with a 1-voxel axis put every point of that axis on the degenerate grid.  Logits are N(0, 1), except head 0, which is
    saturated (+80 on one point, -80 on the others), and head H - 1 (when H > 1), whose logits are all equal."""
    L = len(grids)
    rows = B * sum(x * y * z for x, y, z in grids)
    g = torch.Generator().manual_seed(seed)
    off = torch.randn(rows, H, L, P, 3, generator=g, dtype=torch.float64) * 1.5
    lvl, _, x, y, z = row_coords(grids, B)
    qi = torch.stack([z, y, x], 1).double()
    qdims = torch.tensor([[Z, Y, X] for X, Y, Z in grids], dtype=torch.float64)[lvl]
    pick = torch.rand(rows, H, L, P, 3, generator=g) < planted
    kind = torch.randint(0, len(_KINDS), (rows, H, L, P, 3), generator=g)
    cent = torch.randint(0, 1 << 20, (rows, H, L, P, 3), generator=g)
    for l, (X, Y, Z) in enumerate(grids):
        for a, n in enumerate((Z, Y, X)):
            fref = (qi[:, a] + 0.5) * n / qdims[:, a] - 0.5  # the reference point, un-normalised in level l
            for ki, kn in enumerate(_KINDS):
                m = pick[:, :, l, :, a] & (kind[:, :, l, :, a] == ki)
                if kn.startswith("huge"):
                    val = torch.full((rows, H, P), 1e30 if kn == "huge_hi" else -1e30, dtype=torch.float64)
                elif kn == "centre":
                    val = (cent[:, :, l, :, a] % n).double() - fref[:, None, None]
                else:
                    val = _target(kn, n, 0) - fref[:, None, None].expand(rows, H, P)
                off[:, :, l, :, a] = torch.where(m, val, off[:, :, l, :, a])
    logit = torch.randn(rows, H, L * P, generator=g, dtype=torch.float64)
    hot = torch.arange(rows) % (L * P)
    logit[:, 0] = -80.0
    logit[torch.arange(rows), 0, hot] = 80.0
    if H > 1:
        logit[:, H - 1] = 0.3
    return torch.cat([off.reshape(rows, -1), logit.reshape(rows, -1)], 1).float()


def value_input(grids, B, E, H, head_ld=None, seed=0, pad=0.0):
    """fp32 level-major value rows (rows, H*head_ld), N(0, 1) per level with a per-level offset; the pad columns of a
    padded layout (head_ld > E/H) hold `pad` (NaN: a read of the pad poisons the output)"""
    hd = E // H
    head_ld = hd if head_ld is None else head_ld
    rows = B * sum(x * y * z for x, y, z in grids)
    g = torch.Generator().manual_seed(seed)
    v = torch.full((rows, H, head_ld), pad, dtype=torch.float32)
    v[:, :, :hd] = torch.randn(rows, H, hd, generator=g) + torch.randn(1, H, hd, generator=g)
    return v.reshape(rows, H * head_ld)


def coarse_input(B, Xc, Yc, Zc, C, seed):
    """fp32 (B, Xc, Yc, Zc, C) coarse level of the FPN step, N(0, 1) with a smooth per-voxel offset"""
    g = torch.Generator().manual_seed(seed)
    ramp = torch.linspace(-1, 1, Xc)[:, None, None, None] + torch.linspace(0, 0.5, Yc)[None, :, None, None]
    return torch.randn(B, Xc, Yc, Zc, C, generator=g) + ramp + math.pi / 10


# ------------------------------------------------------------------------------------------------ the GPU test's cases
# occ_ms_deform_attn: (grids coarse -> fine, strides, E, H, B, head_ld values to run)
MSDA_CASES = [
    ([(7, 7, 1), (13, 13, 2), (25, 25, 4)], (12, 6, 3), 192, 8, 1, (32, 24)),  # hd 24, padded and packed heads
    ([(9, 6, 3)], (4,), 32, 4, 3, (8,)),                                      # L = 1, hd 8 (64 threads), Z = 3
    ([(3, 5, 2), (6, 10, 4)], (8, 4), 64, 2, 2, (32,)),                       # L = 2, hd 32 (256 threads)
    ([(2, 2, 1), (4, 3, 2), (8, 6, 4), (16, 12, 8)], (16, 8, 4, 2), 96, 4, 2, (24,)),  # L = 4, 4 passes per patch
    ([(5, 7, 3), (10, 14, 6)], (8, 4), 128, 4, 1, (32,)),                     # Z = 3 and 6: a partial last pass
    ([(3, 2, 2), (6, 4, 3), (12, 8, 6)], (8, 4, 2), 96, 4, 2, (24, 32)),     # the port's shape, B = 2
    ([(25, 25, 2), (50, 50, 4), (100, 100, 8)], (16, 8, 4), 192, 8, 1, (32,)),  # the microbenchmark's 91 250 rows
]

# occ_gn_upsample_add: (B, fine (X, Y, Z), coarse (Xc, Yc, Zc), C, groups)
GN_UP_CASES = [
    (2, (18, 10, 20), (9, 5, 10), 192, 32),     # x2: 3 x 2 x 2 boxes, partial on every axis, cpg 6
    (1, (16, 16, 2), (8, 8, 1), 96, 32),        # x2, cpg 3
    (1, (32, 16, 32), (16, 8, 16), 192, 24),    # x2: two z boxes, cpg 8
    (1, (25, 25, 4), (13, 13, 2), 192, 32),     # general
    (2, (13, 13, 2), (7, 7, 1), 192, 3),        # general, cpg 64
    (1, (16, 12, 3), (8, 6, 2), 96, 32),        # general: x2 in X and Y only
    (2, (5, 4, 3), (5, 4, 3), 1024, 32),        # general: identity size, C4 = 256
    (1, (6, 5, 3), (4, 3, 2), 2048, 32),        # general: the c4 loop runs twice, cpg 64
]

# occ_gn_stats: (B, rows per sample, C, cpg)
GN_STATS_CASES = [
    (1, 49, 192, 6),
    (3, 1250, 192, 6),
    (2, 1, 96, 3),
    (1, 33, 96, 1),       # 96 groups
    (2, 100, 1024, 32),
    (1, 40, 2048, 64),    # more float4 columns than threads
    (1, 64, 256, 256),    # one group
]

# occ_neck_token_prep: grids per level count
TOKEN_GRIDS = {1: [(5, 4, 3)], 3: [(2, 2, 1), (4, 3, 2), (5, 5, 3)], 4: [(1, 1, 1), (2, 3, 1), (4, 5, 2), (7, 6, 3)]}
