"""fp64 restatement of the view transformer's lift-splat kernels (csrc/voxel_pool.cu), one entry point at a time, in
plain torch (any device), plus the input builders of tests/test_gpu_lift_splat.py.

  get_geometry   occ_lss_geometry and the inline geometry of occ_lift_splat_fused, in fp64 from the fp32 camera
                 matrices (3x3, 3x4 and 4x4 intrinsics, 3x3 and 4x4 bda).
  depth_softmax  the depth softmax of occ_lift_prologue / occ_lift_splat_fused, in fp64.
  voxel_ids      the voxel index.  This one stays in fp32, the reference's own arithmetic (oracle.port.voxel_index /
                 kept_mask): which voxel a point lands in is decided by that rounding, so the kernels' ids are compared
                 with it bit for bit, on the kernel's own input geometry.
  pool           the pooled grid in fp64 over a given vox_id (the kernel's own), so every output row is checked whatever
                 the geometry's rounding did.  It also returns sum |w f| and the point count of every voxel.
  check_lists    the per-voxel lists a call leaves in its workspace.

Error bound of the pooled grid.  A voxel v holding n points gets out[v] = sum_p w_p f_p, w_p the depth probability
(1 for materialised rows) and f_p a feature row, both fp32 and taken by the reference exactly as the kernel reads them.
The kernel forms each product once in fp32 (relative error <= u = 2^-24, or an absolute 2^-150 where it underflows)
and adds the n products with n - 1 fp32 additions (two per pair of hops inside a round, one onto the row's partial sum
of earlier rounds; a contraction into an fma only removes roundings).  Whatever the order, the standard bound for a
sum of n rounded products gives |out - ref| <= gamma_n sum_p |w_p f_p| + n 2^-150, gamma_n = n u / (1 - n u), and
gamma_n <= (n + 2) u while n (n + 2) <= 2 / u, i.e. for lists of up to 5 790 points (the GPU test asserts that bound
on n).  So every element must satisfy
    |out - ref| <= (n_v + 2) 2^-24 sum_p |w_p f_p| + n_v 2^-149,
and the tensor as a whole the usual kernel gate, tests/util.assert_close at GATE.  The sum runs in the order of the
voxel's list, which atomicExch builds in whatever order the points arrive: the grid is not bit-reproducible, the bound
holds for every order.

tests/test_cpu_lift_reference.py checks these functions against oracle.port and checks that the GPU test's inputs tell
planted mistakes apart; the `mistake` arguments exist for that check only."""
import numpy as np
import torch

from encoder_ref import case_seed  # one seed rule for every kernel-level test
from oracle import port
from occformer_b200 import synth
from util import assert_close, parity_log

GATE = 5e-5              # kernel vs fp64 (tests/util.assert_close, both criteria)
U = 2.0 ** -24           # unit round-off of fp32
MAX_BOUND_N = 5790       # the largest list length for which gamma_n <= (n + 2) u
HOPS = 4                 # list hops per round of vp_pool_kernel
LF_DG = 8                # depth groups of lift_front_kernel
EXTRA_ROWS = 3           # sentinel rows behind every output

# the model's lift grids and one of 7 x 5 x 3 voxels (dyadic cells): at B = 3, V = 315 is not a multiple of 32, so the
# last warp holds 27 voxels and the last block 2 of its 8 warps
GRIDS = dict(synth.GRIDS, odd=([-1.75, 1.75, 0.5], [-1.25, 1.25, 0.5], [0.0, 1.5, 0.5]))


def grid(name):
    """-> (dx, bx, nx) fp32 as the view transformer holds them, (X, Y, Z)"""
    dx, bx, nx = port.gen_dx_bx(*GRIDS[name])
    return dx, bx, nx, (int(nx[0]), int(nx[1]), int(nx[2]))


def grid_floats(dx, bx, nx):
    """the dx0..nx2 arguments of the entry points"""
    return [float(v) for v in (*dx, *bx, *nx)]


# ------------------------------------------------------------------------------------------------ the arithmetic
def get_geometry(frustum, rots, trans, intrins, post_rots, post_trans, bda):
    """get_geometry in fp64 from fp32 inputs: frustum (..., 3) -> (B, N, P, 3) ego points, P = frustum points"""
    d = lambda t: t.double()  # noqa: E731
    B, N = trans.shape[:2]
    pts = d(frustum).reshape(1, 1, -1, 3) - d(post_trans).view(B, N, 1, 3)
    pts = torch.einsum("bnij,bnpj->bnpi", torch.linalg.inv(d(post_rots)), pts)
    pts = torch.cat((pts[..., :2] * pts[..., 2:3], pts[..., 2:3]), -1)
    K = d(intrins)
    if K.shape[-1] == 4:  # the KITTI shift column, rows 0..2
        pts = pts - K[:, :, None, :3, 3]
    comb = d(rots) @ torch.linalg.inv(K[..., :3, :3])
    pts = torch.einsum("bnij,bnpj->bnpi", comb, pts) + d(trans).view(B, N, 1, 3)
    bd = d(bda)
    out = torch.einsum("bij,bnpj->bnpi", bd[:, :3, :3], pts)
    if bd.shape[-1] == 4:
        out = out + bd[:, None, None, :3, 3]
    return out


def depth_groups(D):
    """the bins [d0, d1) of each of lift_front_kernel's depth groups"""
    dper = -(-D // LF_DG)
    return [(g * dper, min(g * dper + dper, D)) for g in range(LF_DG) if g * dper < D]


def depth_softmax(logits, mistake=None):
    """softmax over dim 1 of (BN, D, ...) in fp64.  mistake "group reads one bin past its end": every depth group but
    the first also counts the bin before it (the previous group's last bin) into the sum."""
    x = logits.double()
    e = (x - x.amax(1, keepdim=True)).exp()
    s = e.sum(1, keepdim=True)
    if mistake == "group reads one bin past its end":
        for d0, _ in depth_groups(x.shape[1])[1:]:
            s = s + e[:, d0 - 1:d0]
    elif mistake is not None:
        raise ValueError(mistake)
    return e / s


INDEX_MISTAKES = ["floor", "<= at the upper bound", "sample 0 for every sample"]


def voxel_ids(geom, dx, bx, nx, XYZ, points_per_batch, mistake=None):
    """vox_id of every point of geom (P, 3) fp32: the linear voxel ((b*X + x)*Y + y)*Z + z of sample
    b = p // points_per_batch, -1 when dropped -- the reference's fp32 index arithmetic (int64, on geom's device)"""
    X, Y, Z = XYZ
    dev = geom.device
    dx, bx, nx = dx.to(dev), bx.to(dev), nx.to(dev)
    if mistake == "floor":
        idx = ((geom - (bx - dx / 2.0)) / dx).floor().long()
    else:
        idx = port.voxel_index(geom, dx, bx)
    if mistake == "<= at the upper bound":
        kept = ((idx >= 0) & (idx <= nx)).all(-1)
    else:
        kept = port.kept_mask(idx, nx)
    b = torch.arange(geom.shape[0], device=dev) // points_per_batch
    if mistake == "sample 0 for every sample":
        b = torch.zeros_like(b)
    elif mistake not in (None, *INDEX_MISTAKES):
        raise ValueError(mistake)
    lin = ((b * X + idx[:, 0]) * Y + idx[:, 1]) * Z + idx[:, 2]
    kept &= (lin >= 0) & (lin < b.max().add(1) * X * Y * Z)  # an index of nx spills into the next row: never past V
    return torch.where(kept, lin, torch.full_like(lin, -1))


def coord_ids(coords, B, XYZ):
    """vox_id of bev_pool's (n, 4) int64 (x, y, z, b) coords: -1 for any coordinate out of range"""
    X, Y, Z = XYZ
    x, y, z, b = coords.unbind(1)
    ok = (x >= 0) & (x < X) & (y >= 0) & (y < Y) & (z >= 0) & (z < Z) & (b >= 0) & (b < B)
    return torch.where(ok, ((b * X + x) * Y + y) * Z + z, torch.full_like(x, -1))


POOL_MISTAKES = [f"drop point {k}" for k in range(1, 6)] + ["a point counted twice", "last partial channel chunk skipped"]


def list_rank(vox):
    """the position of every kept point in its voxel's list, points in ascending order (-1 for dropped points)"""
    keep = vox >= 0
    p = keep.nonzero().flatten()
    v = vox[p]
    order = torch.argsort(v, stable=True)
    cnt = torch.bincount(v, minlength=int(v.max()) + 1 if v.numel() else 1)
    start = torch.cumsum(cnt, 0) - cnt
    rank = torch.full_like(vox, -1)
    rank[p[order]] = torch.arange(p.numel(), device=vox.device) - start[v[order]]
    return rank


def pool(vox, w, rows, feat, V, mistake=None):
    """out[v] = sum over points p with vox[p] = v of w[p] * feat[rows[p]] in fp64 (w None: 1) ->
    (out (V, C), sum |w f| (V, C), count (V,)), on feat's device, in chunks of 2^24 elements"""
    dev = feat.device
    vox, rows = vox.to(dev), rows.to(dev)
    C = feat.shape[1]
    p = (vox >= 0).nonzero().flatten()
    if mistake is not None and mistake.startswith("drop point"):
        k = int(mistake.split()[-1])
        p = p[list_rank(vox)[p] != k - 1]
    elif mistake == "a point counted twice":
        p = torch.cat([p, p[list_rank(vox)[p] == 0]])
    elif mistake not in (None, "last partial channel chunk skipped"):
        raise ValueError(mistake)
    out = torch.zeros(V, C, dtype=torch.float64, device=dev)
    ab = torch.zeros_like(out)
    step = max(1, (1 << 24) // C)
    for s in range(0, p.numel(), step):
        pp = p[s:s + step]
        t = feat[rows[pp]].double()
        if w is not None:
            t = t * w.reshape(-1).to(dev)[pp].double()[:, None]
        out.index_add_(0, vox[pp], t)
        ab.index_add_(0, vox[pp], t.abs())
    if mistake == "last partial channel chunk skipped" and C // 4 > 32 and (C // 4) % 32:
        out[:, (C // 4) // 32 * 128:] = 0
    count = torch.bincount(vox[vox >= 0], minlength=V)
    return out, ab, count


def bound(ab, count):
    """the per-element bound of the module docstring"""
    n = count.double()[:, None]
    return (n + 2) * U * ab + n * 2.0 ** -149


def assert_pooled(out, vox, w, rows, feat, V, what):
    """a kernel's pooled grid out (V, C) against pool() over vox (the kernel's own ids): every element within bound(),
    the occupied rows at GATE (tests/util.assert_close), the empty rows +0.0 -> the reference's counts"""
    want, ab, count = pool(vox, w, rows, feat, V)
    assert int(count.max()) <= MAX_BOUND_N, f"{what}: a list of {int(count.max())} points is past the bound's range"
    nv = int(((out.double() - want).abs() > bound(ab, count)).sum())
    parity_log(f"[bound] {what}: {nv} elements past (n + 2) u sum |w f|, longest list {int(count.max())}")
    assert nv == 0, f"{what}: {nv} elements past the per-voxel bound"
    occ = count > 0
    assert bool((out[~occ].view(torch.int32) == 0).all()), f"{what}: an empty voxel's row is not +0.0"
    assert_close(out[occ], want[occ], GATE, what)
    return count


def s32(t):
    """the values an fp32 tensor keeps in the S32 split format: bf16 hi + bf16 lo of the remainder (fp64)"""
    f = t.float()
    hi = f.bfloat16().float()
    return hi.double() + (f - hi).bfloat16().double()


def twin(out, count, mistake=None):
    """the decoded S32 twin of a pooled grid.  mistake "twin of a multi-round voxel not written": the rows of voxels
    with more than HOPS points stay zero (the twin row is written only in a voxel's last round)"""
    t = s32(out)
    if mistake == "twin of a multi-round voxel not written":
        t[count.to(t.device) > HOPS] = 0
    elif mistake is not None:
        raise ValueError(mistake)
    return t


def lift_rows(B, N, D, HW):
    """the feature row bn * HW + pix of every frustum point p = (bn * D + d) * HW + pix (fused lift)"""
    p = torch.arange(B * N * D * HW)
    return (p // (D * HW)) * HW + p % HW


# ------------------------------------------------------------------------------------------------ list walk
def check_lists(vox, counts, head, nxt):
    """the per-voxel lists of a call (1-based point ids, 0 = end / empty): counts == bincount(vox), and walking head /
    next visits every kept point exactly once, inside its own voxel (any device)"""
    vox, counts, head, nxt = (t.long() for t in (vox, counts, head, nxt))
    kept = vox >= 0
    assert torch.equal(counts, torch.bincount(vox[kept], minlength=counts.numel())), "counts differ from the bincount"
    assert torch.equal(head != 0, counts != 0), "list heads and counts disagree on which voxels are occupied"
    visited = torch.zeros(vox.numel(), dtype=torch.long, device=vox.device)
    cur = head.clone()
    vidx = torch.arange(head.numel(), device=vox.device)
    nxt0 = torch.cat([nxt, torch.zeros(1, dtype=torch.long, device=vox.device)])
    for _ in range(int(counts.max()) + 1 if counts.numel() else 1):
        live = cur != 0
        if not bool(live.any()):
            break
        p = cur[live] - 1
        assert torch.equal(vox[p], vidx[live]), "a list contains a point of another voxel"
        visited[p] += 1
        cur = torch.where(live, nxt0[(cur - 1).clamp(min=-1)], cur)
    assert not bool((cur != 0).any()), "a list is longer than its voxel's count"
    assert torch.equal(visited, kept.long()), "kept points and list membership differ"


def check_bookkeeping(ws, gf, kept, B, X, Y, Z):
    """a workspace's vox_id / counts / lists against the reference's index math (gf (P, 4) int64 (x, y, z, b), kept
    mask) exactly, and its counts against the interval lengths of bev_pool in the reference's own rank order"""
    vox = ws.vox_id.cpu().long()
    ref_lin = ((gf[:, 3] * X + gf[:, 0]) * Y + gf[:, 1]) * Z + gf[:, 2]
    ref_vox = torch.where(kept, ref_lin, torch.full_like(ref_lin, -1))
    assert torch.equal(vox, ref_vox), f"voxel ids differ at {(vox != ref_vox).sum()} points"
    counts = ws.counts.cpu().long()
    assert int(counts.sum()) == int(kept.sum())
    # interval bookkeeping in the reference's own rank order (bev_pool.py:86-93 / QuickCumsumCuda :40-45)
    uniq, lens = port.bev_pool_bookkeeping(gf[kept], B, Z, X, Y)
    nzv = torch.nonzero(counts).flatten()
    b = nzv // (X * Y * Z); r = nzv % (X * Y * Z); x = r // (Y * Z); y = (r // Z) % Y; z = r % Z
    my_ranks = x * (Y * Z * B) + y * (Z * B) + z * B + b
    order = my_ranks.argsort()
    assert torch.equal(my_ranks[order], uniq) and torch.equal(counts[nzv][order], lens)
    check_lists(vox, counts, ws.head.cpu(), ws.next.cpu())


# ------------------------------------------------------------------------------------------------ inputs
LONG = 601                               # the long list: 150 full rounds and one hop
MIXED = [1, 2, 3, 4, 5, 8, 9, 0]         # lane l of the mixed warp holds MIXED[l % 8] points
SMALL = [1, 2, 0]                        # the small warp: no lane beyond two points (the any_gt2 branch not taken)
TAIL = [3, 0, 1, 5, 2]                   # the last warp (partial when V % 32 != 0); its last voxel holds 2


def planted_counts(V):
    """{voxel id: points} of the planted layout over the whole grid: warp 0 mixed, warp 1 empty, warp 2 small, warp 3
    one lane of LONG points and 31 lanes of one, the last warp TAIL[l % 5] and 2 in the grid's last voxel"""
    want = {}
    for lane in range(32):
        want[lane] = MIXED[lane % 8]
        want[64 + lane] = SMALL[lane % 3]
        want[96 + lane] = LONG if lane == 0 else 1
    last = (V - 1) // 32 * 32
    assert last >= 128, f"grid of {V} voxels too small for the planted warps"
    for v in range(last, V):
        want[v] = TAIL[(v - last) % 5]
    want[V - 1] = 2
    return {v: n for v, n in want.items() if n}


def planted_warps(V):
    """the voxel ids of the planted warps (no other point may land in them)"""
    last = (V - 1) // 32 * 32
    return torch.cat([torch.arange(0, 128), torch.arange(last, V)])


def _center(i, a, dx, bx):
    """an fp32 coordinate in the middle of cell i of axis a"""
    o = float(bx[a]) - float(dx[a]) / 2.0
    return np.float32(o + (i + 0.5) * float(dx[a]))


def _voxel_point(v, dx, bx, XYZ):
    X, Y, Z = XYZ
    z = v % Z; y = (v // Z) % Y; x = (v // (Y * Z)) % X
    return [_center(x, 0, dx, bx), _center(y, 1, dx, bx), _center(z, 2, dx, bx)]


def edge_values(a, dx, bx, nx):
    """fp32 coordinates along axis a where the index rules bite: every cell edge computed in fp32 and one ulp either
    side of it, the band (-1, 0) of the index (truncated to 0: kept), exactly nx dx past the origin and one ulp below,
    +-1e30 and +-inf"""
    f = np.float32
    o = f(f(bx[a]) - f(dx[a]) / f(2))
    d = f(dx[a])
    vals = []
    for i in range(int(nx[a]) + 1):
        e = f(o + f(i) * d)
        vals += [e, np.nextafter(e, f(-np.inf)), np.nextafter(e, f(np.inf))]
    top = f(o + f(nx[a]) * d)
    vals += [f(o - f(0.5) * d), f(o - f(0.999) * d), np.nextafter(o, f(-np.inf)), top, np.nextafter(top, f(-np.inf)),
             f(1e30), f(-1e30), f(np.inf), f(-np.inf)]
    return vals


def pool_case(name, B, Pb, seed):
    """geometry of B samples of Pb points each, fp32 (B * Pb, 3): the planted layout (planted_counts), at cell centres,
    in random slots of each voxel's sample; the edge points of every axis (edge_values, the other two axes at the
    middle cell) in sample B - 1; the other slots random voxels outside the planted warps (three in four) or points
    far outside the grid.  -> (geom, planted counts)"""
    dx, bx, nx, XYZ = grid(name)
    X, Y, Z = XYZ
    Vb = X * Y * Z
    V = B * Vb
    g = torch.Generator().manual_seed(seed)
    want = planted_counts(V)
    slots = [torch.randperm(Pb, generator=g).tolist() for _ in range(B)]
    used = [0] * B
    geom = np.zeros((B * Pb, 3), dtype=np.float32)

    def put(b, xyz):
        assert used[b] < Pb, f"sample {b}: more than {Pb} points"
        geom[b * Pb + slots[b][used[b]]] = xyz
        used[b] += 1

    for v, n in want.items():
        for _ in range(n):
            put(v // Vb, _voxel_point(v, dx, bx, XYZ))
    mid = [_center(X // 2, 0, dx, bx), _center(Y // 2, 1, dx, bx), _center(Z // 2, 2, dx, bx)]
    for a in range(3):
        for e in edge_values(a, dx, bx, nx):
            xyz = list(mid)
            xyz[a] = e
            put(B - 1, xyz)
    banned = torch.zeros(V, dtype=torch.bool)
    banned[planted_warps(V)] = True
    for b in range(B):
        free = (~banned[b * Vb:(b + 1) * Vb]).nonzero().flatten() + b * Vb
        while used[b] < Pb:
            if free.numel() and int(torch.randint(4, (1,), generator=g)) < 3:
                put(b, _voxel_point(int(free[int(torch.randint(free.numel(), (1,), generator=g))]), dx, bx, XYZ))
            else:
                put(b, [mid[0], mid[1], np.float32(float(bx[2]) - 50.0)])
    return torch.from_numpy(geom), want


def weights_and_features(P, R, C, seed):
    """planted cases: weights in [0.5, 1] (P,), features N(0, 1) (R, C) -- a dropped or doubled point moves its voxel
    by O(1)"""
    g = torch.Generator().manual_seed(seed)
    return 0.5 + 0.5 * torch.rand(P, generator=g), torch.randn(R, C, generator=g)


def special_pixels(BN, HW):
    """(camera, pixel, kind) of the planted depth distributions: one-hot (one bin 100 above the others), uniform, every
    logit offset by 1e3"""
    return [(0, 0, "onehot"), (1 % BN, min(1, HW - 1), "uniform"), (2 % BN, HW - 1, "offset"), (3 % BN, HW // 2, "onehot")]


def front_case(B, N, D, fH, fW, C, seed):
    """inputs of occ_lift_splat_fused: (logits (BN, D, fH, fW) 3 randn with special_pixels, img_feat (BN, C, fH, fW),
    frustum (D, fH, fW, 3) of a 256 x 704 image with bins 2 + 0.5 d, cameras: nusc cameras with a distinct
    intrinsics, post_rots (rotated, scaled) and bda per camera / sample)"""
    g = torch.Generator().manual_seed(seed)
    BN, HW = B * N, fH * fW
    logits = 3.0 * torch.randn(BN, D, HW, generator=g)
    for bn, pix, kind in special_pixels(BN, HW):
        if kind == "onehot":
            logits[bn, :, pix] = 0.0
            logits[bn, (D - 1) if pix else D // 2, pix] = 100.0
        elif kind == "uniform":
            logits[bn, :, pix] = 0.7
        else:
            logits[bn, :, pix] += 1e3
    feat = torch.randn(BN, C, fH, fW, generator=g)
    ds = torch.arange(D, dtype=torch.float32).mul(0.5).add(2.0).view(D, 1, 1).expand(D, fH, fW)
    xs = torch.linspace(0, 703, fW).view(1, 1, fW).expand(D, fH, fW)
    ys = torch.linspace(0, 255, fH).view(1, fH, 1).expand(D, fH, fW)
    frustum = torch.stack((xs, ys, ds), -1).contiguous()
    return logits.view(BN, D, fH, fW), feat, frustum, cameras(B, N, 3, 3, seed)


def cameras(B, N, intrin_cols, bda_dim, seed, intrin_rows=3):
    """nuScenes-like cameras with a distinct matrix per camera and a distinct bda per sample: intrinsics 3 x 3, 3 x 4
    (shift column) or 4 x 4 (KITTI P2), post_rots a small rotation and resize, bda a yaw, flip-free scale and (4 x 4)
    translation"""
    g = torch.Generator().manual_seed(seed)
    cams = synth.nusc_cameras(B, N)
    r = lambda *s: torch.rand(*s, generator=g) - 0.5  # noqa: E731
    K = torch.zeros(B, N, intrin_rows, intrin_cols)
    K[..., :3, :3] = cams["intrins"] * (1 + 0.05 * r(B, N, 1, 1))
    K[..., 2, 2] = 1.0
    if intrin_cols == 4:
        K[..., :3, 3] = torch.tensor([45.76, -0.35, 0.005]) + r(B, N, 3)
        if intrin_rows == 4:
            K[..., 3, 3] = 1.0
    cams["intrins"] = K
    a = 0.1 * r(B, N)
    s = 0.44 * (1 + 0.1 * r(B, N))
    pr = torch.zeros(B, N, 3, 3)
    pr[..., 0, 0], pr[..., 0, 1], pr[..., 1, 0], pr[..., 1, 1] = s * a.cos(), -s * a.sin(), s * a.sin(), s * a.cos()
    pr[..., 2, 2] = 1.0
    cams["post_rots"] = pr
    cams["post_trans"] = cams["post_trans"] + 5 * r(B, N, 3)
    cams["trans"] = cams["trans"] + 0.1 * r(B, N, 3)
    yaw = 0.2 * r(B)
    bda = torch.zeros(B, bda_dim, bda_dim)
    bda[:, 0, 0], bda[:, 0, 1], bda[:, 1, 0], bda[:, 1, 1] = yaw.cos(), -yaw.sin(), yaw.sin(), yaw.cos()
    bda[:, :3, :3] *= (1 + 0.05 * r(B)).view(B, 1, 1)
    bda[:, 2, 2] = 1.0 + 0.05 * r(B)
    if bda_dim == 4:
        bda[:, :3, 3] = r(B, 3)
        bda[:, 3, 3] = 1.0
    return {k: v.float().contiguous() for k, v in cams.items()}


def identity_cameras(B, N):
    """rots = post_rots = K = bda = I, trans = post_trans = 0: a frustum point (x, y, 1) maps exactly to (x, y, 1)"""
    eye = lambda n, *lead: torch.eye(n).expand(*lead, n, n).contiguous()  # noqa: E731
    return dict(rots=eye(3, B, N), trans=torch.zeros(B, N, 3), intrins=eye(3, B, N), post_rots=eye(3, B, N),
                post_trans=torch.zeros(B, N, 3), bda=eye(3, B))


def identity_frustum(name, D, HW, seed):
    """(D * HW, 3) frustum points (x, y, 1) of the planted column layout of the `name` grid for identity cameras: every
    point's ego point is itself, so all of them land in the z-layer of 1.0.  Column c (x, y) of that layer takes
    FRUSTUM_COUNTS[c % 9] points (the first column LONG - 1, so with N = 1 one list spans 150 rounds); the rest of the
    slots are (x, y) far outside the grid"""
    dx, bx, nx, (X, Y, Z) = grid(name)
    iz = int((1.0 - (float(bx[2]) - float(dx[2]) / 2)) / float(dx[2]))
    assert 0 <= iz < Z
    g = torch.Generator().manual_seed(seed)
    slots = torch.randperm(D * HW, generator=g).tolist()
    fr = np.zeros((D * HW, 3), dtype=np.float32)
    fr[:, 0], fr[:, 1], fr[:, 2] = -1e4, -1e4, 1.0
    k = 0
    for c in range(X * Y):
        n = LONG - 1 if c == 0 else FRUSTUM_COUNTS[c % 9]
        for _ in range(n):
            assert k < len(slots), "frustum too small for the planted columns"
            fr[slots[k], :2] = [_center(c // Y, 0, dx, bx), _center(c % Y, 1, dx, bx)]
            k += 1
    return torch.from_numpy(fr)


FRUSTUM_COUNTS = [1, 2, 3, 4, 5, 8, 9, 0, 1]


# ------------------------------------------------------------------------------------------------ the GPU test's cases
POOL_GRIDS = [("pr1", 2), ("nusc_200", 2), ("kitti", 2), ("odd", 3)]   # (grid, B)
POOL_C = [4, 8, 36, 124, 128, 132, 260, 516]
POOL_N, POOL_D, POOL_HW = 2, 9, 250          # Pb = 4 500 points per sample: D * HW not a power of two
FRONT_D = [1, 7, 8, 9, 59, 112, 256]
FRONT_HW = {1: (1, 1), 31: (1, 31), 32: (2, 16), 33: (3, 11), 704: (16, 44)}   # HW -> (fH, fW)
MISTAKE_CASE = ("pr1", 2, 132)              # pooling mistakes: grid, B, C (C / 4 = 33: one partial channel chunk)
FRONT_MISTAKE_HW = 704


def seed_of(name, *case):
    """one fixed seed per case: a grid name and integers"""
    return case_seed(sorted(GRIDS).index(name), *case)
