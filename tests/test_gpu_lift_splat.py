"""The view transformer's lift-splat kernels (csrc/voxel_pool.cu) one entry point at a time, through ops._call, against
the fp64 reference of tests/lift_ref.py: occ_lss_geometry, occ_lift_prologue, occ_lift_splat_fused, occ_lift_splat,
occ_voxel_pool_geom and occ_bev_pool.  tests/test_cpu_lift_reference.py checks the reference, and that these inputs tell
planted mistakes apart.

Every call writes into SENTINEL buffers with spare rows behind the output and uses a workspace of its own (no state
shared with other tests).  Checked bit for bit: voxel ids and counts against the reference's fp32 index math on the
kernel's own input geometry (planted lists of 1, 2, 3, 4, 5, 8, 9 and 601 points, one long list in a warp of single
points, cell edges and one ulp either side, the (-1, 0) band, nx dx, +-1e30 and +-inf), the fused kernel's ids against
occ_lss_geometry + occ_lift_splat's index, the NHWC features, the S32 twin against ops.to_split of the grid, launch
counts, rejected arguments.  Within the bound of lift_ref: the pooled grid against fp64 pooling over the kernel's own
vox_id, element by element and at GATE; the depth softmax and the geometry at GATE.  The lists are walked: every kept
point once, inside its own voxel.  The grid is not bit-reproducible (list order comes from atomicExch), so repeats and
graph replay are held to the bound, their ids and counts to the bit."""
import functools

import pytest
import torch

import lift_ref as ref
from occformer_b200 import ops, synth
from oracle import port
from util import SENTINEL, assert_close, graph_replay, launches, parity_log, rejected, same_bits, sentinel, untouched

pytestmark = pytest.mark.gpu

GATE = ref.GATE
EXTRA = ref.EXTRA_ROWS


def _ws(P, B, X, Y, Z, dev, short=0):
    nbytes = ops.lib().occ_voxel_pool_workspace_bytes(P, B, X, Y, Z) - short
    return ops.VoxelPoolWorkspace(torch.zeros(nbytes, dtype=torch.uint8, device=dev), P, B, X, Y, Z)


def _buf(rows, cols, dev):
    """(buffer, its first `rows` rows): SENTINEL everywhere, EXTRA rows behind the output"""
    b = sentinel(rows + EXTRA, cols, dev)
    return b, b[:rows]


def _cam_args(cams, dev):
    """rots, trans, intrins, rows, cols, post_rots, post_trans, bda, bda_dim as the entry points take them"""
    c = {k: v.float().contiguous().to(dev) for k, v in cams.items()}
    k = c["intrins"]
    return [c["rots"], c["trans"], k, k.shape[-2], k.shape[-1], c["post_rots"], c["post_trans"], c["bda"],
            c["bda"].shape[-1]]


def _judge_grid(out, buf, vox, w, rows, feat, V, what):
    """nothing written past the output, nothing left of the SENTINEL inside it, and lift_ref.assert_pooled ->
    the reference's counts"""
    untouched(buf[V:], f"{what}: rows past the output")
    assert not bool((out.view(torch.int32) == SENTINEL).any()), f"{what}: output rows left unwritten"
    return ref.assert_pooled(out, vox, w, rows, feat, V, what)


# ------------------------------------------------------------------------------------------------ geometry
@pytest.mark.parametrize("intrin_rows,intrin_cols", [(3, 3), (3, 4), (4, 4)])
@pytest.mark.parametrize("bda_dim", [3, 4])
def test_lss_geometry_against_fp64(cuda, intrin_rows, intrin_cols, bda_dim):
    """B = 3, N = 2: a distinct intrinsics, post_rots (rotation and resize) and post_trans per camera, a distinct bda
    per sample"""
    B, N = 3, 2
    _, _, frustum, _ = ref.front_case(1, 1, 59, 16, 44, 4, 0)
    cams = ref.cameras(B, N, intrin_cols, bda_dim, ref.case_seed(intrin_rows, intrin_cols, bda_dim), intrin_rows)
    P = frustum.numel() // 3
    buf, geom = _buf(B * N * P, 3, cuda)
    n = launches("occ_lss_geometry", frustum.to(cuda), P, *_cam_args(cams, cuda), B, N, geom)
    assert n == 1, f"{n} launches"
    untouched(buf[B * N * P:], "rows past the geometry")
    want = ref.get_geometry(frustum, **cams).reshape(-1, 3)
    assert_close(geom, want, GATE, f"lss_geometry intrins {intrin_rows}x{intrin_cols} bda {bda_dim}")


# ------------------------------------------------------------------------------------------------ front kernel
def _front(cuda, B, N, D, HW, C, seed, grid_name="nusc_200", strided=False, cams=None, logits=None, frustum=None):
    """occ_lift_splat_fused into sentinel buffers -> dict of its outputs, workspace and inputs"""
    fH, fW = ref.FRONT_HW.get(HW, (1, HW))
    lg, feat, fr, cm = ref.front_case(B, N, D, fH, fW, C, seed)
    cams = cm if cams is None else cams
    lg = lg if logits is None else logits
    fr = fr if frustum is None else frustum
    dx, bx, nx, (X, Y, Z) = ref.grid(grid_name)
    BN, V = B * N, B * X * Y * Z
    x = torch.cat([lg, feat], 1).to(cuda)
    if strided:  # channel slices of one (BN, D + C, fH, fW) map, passed without a copy
        lp, ls, fp, fs = x.data_ptr(), (D + C) * HW, x[:, D:].data_ptr(), (D + C) * HW
    else:
        lp, fp = x[:, :D].contiguous(), x[:, D:].contiguous()
        ls, fs = D * HW, C * HW
    pbuf, prob = _buf(BN * D, HW, cuda)
    fbuf, feat_cl = _buf(BN * HW, C, cuda)
    obuf, out = _buf(V, C, cuda)
    sbuf, out_s = _buf(V, C, cuda) if C % 32 == 0 else (None, None)
    ws = _ws(BN * D * HW, B, X, Y, Z, cuda)
    n = launches("occ_lift_splat_fused", lp, ls, fp, fs, fr.to(cuda).contiguous(), *_cam_args(cams, cuda), prob, feat_cl,
                 out, out_s, B, N, D, HW, C, *ref.grid_floats(dx, bx, nx), X, Y, Z, ws.buf, ws.nbytes)
    assert n == 3, f"{n} launches"
    untouched(pbuf[BN * D:], "rows past depth_prob")
    untouched(fbuf[BN * HW:], "rows past feat_cl")
    return dict(prob=prob, feat_cl=feat_cl, out=out, obuf=obuf, out_s=out_s, sbuf=sbuf, ws=ws, logits=lg, feat=feat,
                frustum=fr, cams=cams, grid=(dx, bx, nx, (X, Y, Z)), V=V)


@pytest.mark.parametrize("HW", sorted(ref.FRONT_HW))
@pytest.mark.parametrize("D", ref.FRONT_D)
def test_lift_front_kernel(cuda, D, HW):
    """D < 8, not a multiple of 8, 256 bins; HW around one 32-pixel tile and the R50 map; logits / features contiguous
    and as channel slices of one map.  The fused kernel's ids and counts are those of occ_lss_geometry followed by
    occ_lift_splat's index on the same cameras: its inline geometry is the same arithmetic."""
    B, N, C = 2, 2, 40
    seed = ref.case_seed(D, HW)
    r = _front(cuda, B, N, D, HW, C, seed)
    BN, case = B * N, f"D{D} HW{HW}"
    want = ref.depth_softmax(r["logits"]).to(cuda)
    prob = r["prob"].view(BN, D, HW)
    assert_close(prob, want.view(BN, D, HW), GATE, f"fused depth_prob {case}")
    for bn, pix, kind in ref.special_pixels(BN, HW):
        assert_close(prob[bn, :, pix], want.view(BN, D, HW)[bn, :, pix], GATE, f"fused depth_prob {case} {kind} pixel")
    feat_nhwc = r["feat"].to(cuda).permute(0, 2, 3, 1).reshape(BN * HW, C)
    same_bits(r["feat_cl"], feat_nhwc, f"feat_cl {case}")
    ws = r["ws"]
    dx, bx, nx, (X, Y, Z) = r["grid"]
    V = r["V"]
    ref.check_lists(ws.vox_id, ws.counts, ws.head, ws.next)
    _judge_grid(r["out"], r["obuf"], ws.vox_id.long(), r["prob"], ref.lift_rows(B, N, D, HW), r["feat_cl"], V,
                f"fused grid {case}")
    # the same cameras through occ_lss_geometry + occ_lift_splat
    P = D * HW
    geom = torch.empty(BN * P, 3, device=cuda)
    ops._call("occ_lss_geometry", r["frustum"].to(cuda).contiguous(), P, *_cam_args(r["cams"], cuda), B, N, geom)
    ws2 = _ws(BN * P, B, X, Y, Z, cuda)
    out2 = torch.empty(V, C, device=cuda)
    n = launches("occ_lift_splat", r["prob"], r["feat_cl"], geom, out2, None, B, N, D, HW, C,
                 *ref.grid_floats(dx, bx, nx), X, Y, Z, ws2.buf, ws2.nbytes)
    assert n == 3, f"{n} launches"
    same_bits(ws.vox_id, ws2.vox_id, f"fused ids vs occ_lss_geometry + occ_lift_splat {case}")
    same_bits(ws.counts, ws2.counts, f"fused counts vs occ_lss_geometry + occ_lift_splat {case}")
    same_bits(ws.vox_id.long(), ref.voxel_ids(geom.cpu(), dx, bx, nx, (X, Y, Z), N * P).to(cuda).int().long(),
              f"ids vs the fp32 index math {case}")
    # the strided layout: the same bits
    s = _front(cuda, B, N, D, HW, C, seed, strided=True)
    for k in ("prob", "feat_cl"):
        same_bits(s[k], r[k], f"strided {k} {case}")
    same_bits(s["ws"].vox_id, ws.vox_id, f"strided ids {case}")
    same_bits(s["ws"].counts, ws.counts, f"strided counts {case}")
    # occ_lift_prologue: the two-kernel softmax + transpose
    pbuf, p2 = _buf(BN * D, HW, cuda)
    fbuf, f2 = _buf(BN * HW, C, cuda)
    n = launches("occ_lift_prologue", r["logits"].to(cuda).contiguous(), r["feat"].to(cuda).contiguous(), p2, f2, BN, D,
                 C, HW)
    assert n == 2, f"{n} launches"
    untouched(pbuf[BN * D:], "rows past the prologue's depth_prob")
    untouched(fbuf[BN * HW:], "rows past the prologue's feat_cl")
    assert_close(p2.view(BN, D, HW), want.view(BN, D, HW), GATE, f"prologue depth_prob {case}")
    same_bits(f2, feat_nhwc, f"prologue feat_cl {case}")


@pytest.mark.parametrize("C", [36, 128])
def test_lift_splat_fused_planted_lists(cuda, C):
    """identity cameras: the frustum is the geometry, so planted lists (1 .. 9 and 600 points) reach the fused path;
    the odd grid (V % 32 != 0); the S32 twin (C = 128) bit for bit, multi-round rows included"""
    B, N, D, HW = 2, 1, ref.POOL_D, 100
    fr = ref.identity_frustum("odd", D, HW, 3)
    g = torch.Generator().manual_seed(ref.case_seed(C))
    logits = 0.3 * torch.randn(B * N, D, 1, HW, generator=g)   # weights near 1 / D: no point is negligible
    r = _front(cuda, B, N, D, HW, C, ref.case_seed(C, 1), grid_name="odd", cams=ref.identity_cameras(B, N),
               logits=logits, frustum=fr)
    dx, bx, nx, XYZ = r["grid"]
    ws = r["ws"]
    want_ids = ref.voxel_ids(fr.repeat(B * N, 1), dx, bx, nx, XYZ, N * D * HW)
    same_bits(ws.vox_id.long().cpu(), want_ids, "fused ids vs the fp32 index math")
    ref.check_lists(ws.vox_id, ws.counts, ws.head, ws.next)
    count = _judge_grid(r["out"], r["obuf"], ws.vox_id.long(), r["prob"], ref.lift_rows(B, N, D, HW), r["feat_cl"],
                        r["V"], f"fused planted grid C{C}")
    assert int(count.max()) == ref.LONG - 1
    if r["out_s"] is not None:
        untouched(r["sbuf"][r["V"]:], "rows past the twin")
        same_bits(r["out_s"], ops.to_split(r["out"]), "S32 twin of the fused grid")


# ------------------------------------------------------------------------------------------------ pooling
@functools.lru_cache(maxsize=None)
def _pool_case(name, B):
    Pb = ref.POOL_N * ref.POOL_D * ref.POOL_HW
    geom, _ = ref.pool_case(name, B, Pb, ref.seed_of(name, B))
    dx, bx, nx, XYZ = ref.grid(name)
    return geom, ref.voxel_ids(geom, dx, bx, nx, XYZ, Pb), Pb


def _oob_coords(B, XYZ, n, seed):
    """n (x, y, z, b) rows with exactly one coordinate out of range: -1 or the extent on each axis, b = B or -1"""
    X, Y, Z = XYZ
    g = torch.Generator().manual_seed(seed)
    c = torch.stack([torch.randint(X, (n,), generator=g), torch.randint(Y, (n,), generator=g),
                     torch.randint(Z, (n,), generator=g), torch.randint(B, (n,), generator=g)], 1)
    bad = torch.tensor([-1, X, -1, Y, -1, Z, -1, B])
    i = torch.arange(n)
    c[i, (i % 8) // 2] = bad[i % 8]
    return c


def _pool_cases():
    cs = [(name, B, C) for name, B in ref.POOL_GRIDS if name in ("pr1", "odd") for C in ref.POOL_C]
    return cs + [("nusc_200", 2, 4), ("nusc_200", 2, 128), ("kitti", 2, 36), ("kitti", 2, 260)]


@pytest.mark.parametrize("mode", ["lift", "geom", "coords"])
@pytest.mark.parametrize("name,B,C", _pool_cases())
def test_pooling(cuda, mode, name, B, C):
    """occ_lift_splat (lift: w = depth, rows of feat_cl), occ_voxel_pool_geom (materialised rows) and occ_bev_pool
    (coords of the kept points plus rows out of range on every axis and b >= B) on the planted layout and edge
    geometry"""
    geom, want_ids, Pb = _pool_case(name, B)
    dx, bx, nx, (X, Y, Z) = ref.grid(name)
    V, P = B * X * Y * Z, B * Pb
    N, D, HW = ref.POOL_N, ref.POOL_D, ref.POOL_HW
    case = f"{mode} {name} B{B} C{C}"
    fl = ref.grid_floats(dx, bx, nx)
    obuf, out = _buf(V, C, cuda)
    if mode == "lift":
        w, feat = ref.weights_and_features(P, B * N * HW, C, ref.seed_of(name, B, C))
        rows = ref.lift_rows(B, N, D, HW)
        sbuf, out_s = _buf(V, C, cuda) if C % 32 == 0 else (None, None)
        ws = _ws(P, B, X, Y, Z, cuda)
        w, feat = w.to(cuda), feat.to(cuda)
        n = launches("occ_lift_splat", w, feat, geom.to(cuda), out, out_s, B, N, D, HW, C, *fl, X, Y, Z, ws.buf,
                     ws.nbytes)
    elif mode == "geom":
        w, (_, feat) = None, ref.weights_and_features(P, P, C, ref.seed_of(name, B, C))
        rows, feat = torch.arange(P), feat.to(cuda)
        ws = _ws(P, B, X, Y, Z, cuda)
        n = launches("occ_voxel_pool_geom", feat, geom.to(cuda), out, B, Pb, C, *fl, X, Y, Z, ws.buf, ws.nbytes)
    else:
        kept = want_ids[want_ids >= 0]
        coords = torch.stack([(kept // (Y * Z)) % X, (kept // Z) % Y, kept % Z, kept // (X * Y * Z)], 1)
        coords = torch.cat([coords, _oob_coords(B, (X, Y, Z), 64, ref.seed_of(name, B))])
        perm = torch.randperm(coords.shape[0], generator=torch.Generator().manual_seed(C))
        coords = coords[perm].contiguous()
        want_ids = ref.coord_ids(coords, B, (X, Y, Z))
        m = coords.shape[0]
        w, (_, feat) = None, ref.weights_and_features(m, m, C, ref.seed_of(name, B, C))
        rows, feat = torch.arange(m), feat.to(cuda)
        ws = _ws(m, B, X, Y, Z, cuda)
        n = launches("occ_bev_pool", feat, coords.to(cuda), out, m, C, B, X, Y, Z, ws.buf, ws.nbytes)
    assert n == 3, f"{n} launches"
    same_bits(ws.vox_id.long(), want_ids.to(cuda), f"{case} ids vs the fp32 index math")
    ref.check_lists(ws.vox_id, ws.counts, ws.head, ws.next)
    _judge_grid(out, obuf, ws.vox_id.long(), w, rows, feat, V, case)
    if mode == "lift" and out_s is not None:
        untouched(sbuf[V:], f"{case}: rows past the twin")
        same_bits(out_s, ops.to_split(out), f"{case} S32 twin")


def test_bev_pool_empty(cuda):
    """n = 0: the memset and the pooling kernel (no index launch), every row +0.0"""
    B, X, Y, Z, C = 2, 7, 5, 3, 36
    V = B * X * Y * Z
    obuf, out = _buf(V, C, cuda)
    ws = _ws(0, B, X, Y, Z, cuda)
    n = launches("occ_bev_pool", None, None, out, 0, C, B, X, Y, Z, ws.buf, ws.nbytes)
    assert n == 2, f"{n} launches"
    untouched(obuf[V:], "rows past the output")
    assert bool((out.view(torch.int32) == 0).all())


# ------------------------------------------------------------------------------------------------ full size
def test_full_size_r101(cuda):
    """the nusc_r101 frustum (6 cameras, 112 bins, 56 x 100 pixels: 3 763 200 points, D * HW = 627 200 not a power of
    two), lists of several hundred points, fused path with its twin; the fp64 pooling runs on the device"""
    w = synth.WORKLOADS["nusc_r101"]
    B, N, C = 1, w["cams"], 64
    gc = synth.grid_config(w["grid"])
    frustum = port.create_frustum(w["input_size"], 16, gc["dbound"])
    D, fH, fW = frustum.shape[:3]
    HW = fH * fW
    dd, feat = synth.lift_inputs(B, N, D, fH, fW, C, seed=9)
    dx, bx, nx, (X, Y, Z) = ref.grid(w["grid"])
    V, P = B * X * Y * Z, B * N * D * HW
    assert P == 3763200
    pbuf, prob = _buf(B * N * D, HW, cuda)
    fbuf, feat_cl = _buf(B * N * HW, C, cuda)
    obuf, out = _buf(V, C, cuda)
    sbuf, out_s = _buf(V, C, cuda)
    ws = _ws(P, B, X, Y, Z, cuda)
    cams = synth.workload_cameras("nusc_r101", B)
    torch.cuda.reset_peak_memory_stats()
    m0 = torch.cuda.memory_allocated()
    n = launches("occ_lift_splat_fused", dd.to(cuda), D * HW, feat.to(cuda), C * HW, frustum.to(cuda).contiguous(),
                 *_cam_args(cams, cuda), prob, feat_cl, out, out_s, B, N, D, HW, C, *ref.grid_floats(dx, bx, nx), X, Y,
                 Z, ws.buf, ws.nbytes)
    assert n == 3, f"{n} launches"
    untouched(pbuf[B * N * D:], "rows past depth_prob")
    untouched(fbuf[B * N * HW:], "rows past feat_cl")
    untouched(sbuf[V:], "rows past the twin")
    assert_close(prob.view(B * N, D, HW), ref.depth_softmax(dd.to(cuda)).view(B * N, D, HW), GATE, "r101 depth_prob")
    geom = torch.empty(P, 3, device=cuda)
    ops._call("occ_lss_geometry", frustum.to(cuda).contiguous(), D * HW, *_cam_args(cams, cuda), B, N, geom)
    same_bits(ws.vox_id.long().cpu(), ref.voxel_ids(geom.cpu(), dx, bx, nx, (X, Y, Z), N * D * HW),
              "r101 ids vs the fp32 index math on occ_lss_geometry's points")
    ref.check_lists(ws.vox_id, ws.counts, ws.head, ws.next)
    m1 = torch.cuda.max_memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    count = _judge_grid(out, obuf, ws.vox_id.long(), prob, ref.lift_rows(B, N, D, HW).to(cuda), feat_cl, V,
                        "r101 fused grid")
    same_bits(out_s, ops.to_split(out), "r101 S32 twin")
    ref_mb = (torch.cuda.max_memory_allocated() - torch.cuda.memory_allocated()) / 2 ** 20
    parity_log(f"[r101] {P} points, {int((ws.vox_id >= 0).sum())} kept, {int((count > 0).sum())} occupied voxels, "
               f"max list {int(count.max())}, mean {float(count[count > 0].double().mean()):.1f}; fp64 reference peak "
               f"{ref_mb:.0f} MiB beyond the kernel's buffers ({(m1 - m0) / 2 ** 20:.0f} MiB)")
    assert int(count.max()) >= 100


# ------------------------------------------------------------------------------------------------ repeats, graphs
def test_repeat_and_graph_replay(cuda):
    """ids and counts bit-identical across a repeat and a CUDA-graph replay of the fused call; the grid within the bound
    each time (list order, and so the summation order, may change)"""
    B, N, D, HW, C = 2, 2, 59, 704, 128
    r = _front(cuda, B, N, D, HW, C, 11)
    ws = r["ws"]
    ids, counts = ws.vox_id.clone(), ws.counts.clone()
    s = _front(cuda, B, N, D, HW, C, 11)
    same_bits(s["ws"].vox_id, ids, "repeat ids")
    same_bits(s["ws"].counts, counts, "repeat counts")
    rows = ref.lift_rows(B, N, D, HW)
    _judge_grid(s["out"], s["obuf"], ids.long(), s["prob"], rows, s["feat_cl"], r["V"], "repeat grid")
    dx, bx, nx, (X, Y, Z) = r["grid"]
    x_l = r["logits"].to(cuda).contiguous()
    x_f = r["feat"].to(cuda).contiguous()
    fr = r["frustum"].to(cuda).contiguous()
    cam = _cam_args(r["cams"], cuda)
    g_ws = _ws(B * N * D * HW, B, X, Y, Z, cuda)
    obuf, out = _buf(r["V"], C, cuda)
    _, out_s = _buf(r["V"], C, cuda)
    prob, feat_cl = torch.empty_like(r["prob"]), torch.empty_like(r["feat_cl"])
    graph_replay(lambda: ops._call("occ_lift_splat_fused", x_l, D * HW, x_f, C * HW, fr, *cam, prob, feat_cl, out, out_s,
                                   B, N, D, HW, C, *ref.grid_floats(dx, bx, nx), X, Y, Z, g_ws.buf, g_ws.nbytes),
                 [out, out_s, prob, feat_cl, g_ws.vox_id, g_ws.counts])
    same_bits(g_ws.vox_id, ids, "graph replay ids")
    same_bits(g_ws.counts, counts, "graph replay counts")
    same_bits(prob, r["prob"], "graph replay depth_prob")
    same_bits(feat_cl, r["feat_cl"], "graph replay feat_cl")
    ref.check_lists(g_ws.vox_id, g_ws.counts, g_ws.head, g_ws.next)
    _judge_grid(out, obuf, ids.long(), prob, rows, feat_cl, r["V"], "graph replay grid")
    same_bits(out_s, ops.to_split(out), "graph replay S32 twin")


# ------------------------------------------------------------------------------------------------ rejections
def test_rejections(cuda):
    """each rejected call enqueues nothing and leaves its buffers as they were; the exact workspace size is accepted"""
    B, N, D, HW, X, Y, Z = 1, 1, 4, 8, 7, 5, 3
    dx, bx, nx, _ = ref.grid("odd")
    fl = ref.grid_floats(dx, bx, nx)
    V, P = B * X * Y * Z, B * N * D * HW
    z = lambda *s: torch.zeros(*s, device=cuda)  # noqa: E731
    cams = _cam_args(ref.identity_cameras(B, N), cuda)
    prob, geom, fr = z(B * N * D, HW), z(P, 3), z(D * HW, 3)
    ws, short = _ws(P, B, X, Y, Z, cuda), _ws(P, B, X, Y, Z, cuda, short=1)

    def bufs(C):
        out, twin = sentinel(V, C, cuda), sentinel(V, C, cuda)
        return z(B * N * HW, C), out, twin, z(P, C), z(B * N, C, HW)

    def lift(C, twin_on, w=ws):
        f, out, twin, _, _ = bufs(C)
        return ("occ_lift_splat", prob, f, geom, out, twin if twin_on else None, B, N, D, HW, C, *fl, X, Y, Z, w.buf,
                w.nbytes), (out, twin)

    def fused(C, twin_on=False, D_=D, ls=None, cols=3, bda=3, w=ws):
        f, out, twin, _, img = bufs(C)
        lg = z(B * N, D_, HW)
        cam = list(cams)
        cam[4], cam[8] = cols, bda
        return ("occ_lift_splat_fused", lg, D_ * HW if ls is None else ls, img, C * HW, z(D_ * HW, 3), *cam,
                z(B * N * D_, HW), f, out, twin if twin_on else None, B, N, D_, HW, C, *fl, X, Y, Z, w.buf,
                w.nbytes), (out, twin)

    def pool_geom(C, w=ws):
        _, out, _, rows, _ = bufs(C)
        return ("occ_voxel_pool_geom", rows, geom, out, B, P // B, C, *fl, X, Y, Z, w.buf, w.nbytes), (out,)

    def bev(C, w=ws):
        _, out, _, rows, _ = bufs(C)
        return ("occ_bev_pool", rows, torch.zeros(P, 4, dtype=torch.long, device=cuda), out, P, C, B, X, Y, Z, w.buf,
                w.nbytes), (out,)

    for make in (lift, fused):
        for args, outs in (make(6, False), make(36, True), make(32, False, w=short)):  # C % 4, twin C % 32, 1 byte short
            rejected(*args, buffers=outs)
        args, _ = make(32, False)
        assert launches(*args) == 3                                                  # the exact size
    for make in (pool_geom, bev):
        for args, outs in (make(6), make(32, w=short)):
            rejected(*args, buffers=outs)
        args, _ = make(32)
        assert launches(*args) == 3
    for args, outs in (fused(32, D_=257), fused(32, ls=D * HW - 1), fused(32, cols=5), fused(32, bda=2)):
        rejected(*args, buffers=outs)
    g = sentinel(P, 3, cuda)
    rejected("occ_lss_geometry", fr, D * HW, *cams[:4], 5, *cams[5:], B, N, g, buffers=(g,))   # intrin_cols = 5
    rejected("occ_lss_geometry", fr, D * HW, *cams[:8], 2, B, N, g, buffers=(g,))             # bda_dim = 2
    rejected("occ_lss_geometry", fr, D * HW, *cams, 65536, 1, g, buffers=(g,))                 # B * N > 65535
    assert launches("occ_lss_geometry", fr, D * HW, *cams, B, N, g) == 1
