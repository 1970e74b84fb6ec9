"""CPU suite (-m "not gpu"): oracle vs the reference-generated goldens, the drop-in boundary (registry names,
state_dict keys), host-side logic, and that the C-ABI library loads and exports every declared symbol."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from oracle import port
from occformer_b200 import synth
from util import GOLDEN, assert_close, golden, rel_err

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------ oracle pinned by reference goldens
def test_oracle_voxel_pool_vs_reference_golden():
    gd = golden("voxel_pool_pr1.npz")
    gc = synth.grid_config("pr1")
    frustum = port.create_frustum((128, 128), 16, gc["dbound"])
    geom = port.get_geometry(frustum, **synth.pr1_camera(2))
    assert np.array_equal(gd["geom"], geom.numpy()), "get_geometry restatement differs from the reference"
    dx, bx, nx = port.gen_dx_bx(gc["xbound"], gc["ybound"], gc["zbound"])
    D, fH, fW = frustum.shape[:3]
    dd, feat = synth.lift_inputs(2, 1, D, fH, fW, 32, seed=1)
    vol, prob = port.lift(dd, feat, 2, 1)
    out, gf, kept = port.voxel_pooling(geom, vol, dx, bx, nx)
    dense = out.permute(0, 2, 3, 4, 1)
    idx = torch.from_numpy(gd["nonzero_index"]).long()
    nz = torch.nonzero(dense.abs().sum(-1) != 0)
    assert torch.equal(nz, idx), "set of non-empty voxels differs from the reference"
    rows = dense[idx[:, 0], idx[:, 1], idx[:, 2], idx[:, 3]]
    assert rel_err(rows, torch.from_numpy(gd["nonzero_rows"])) < 2e-6
    assert abs(float(prob.double().sum()) - float(gd["depth_prob_sum"])) < 1e-6


@pytest.mark.parametrize("name,cin,c,stride,shift,grid,seed", [
    ("block_c128_s1_plain", 128, 128, 1, False, (15, 10, 4), 1),
    ("block_c256_s2_shift", 128, 256, 2, True, (15, 10, 4), 2),
    ("block_c128_s1_shift", 128, 128, 1, True, (9, 16, 2), 3)])
def test_oracle_block_vs_reference_golden(name, cin, c, stride, shift, grid, seed):
    g = torch.Generator().manual_seed(seed)
    sd = port.make_block_state(cin, c, stride, g)
    x = synth.encoder_input(1, cin, *grid, seed=seed + 100)
    out = port.dualpath_block(x, sd, "", stride, shift)
    assert rel_err(out, torch.from_numpy(golden(name + ".npz")["out"])) < 1e-5


def test_oracle_head_vs_reference_golden():
    gd = golden("head_nusc.npz")
    E, Q, K, L = 96, 12, 17, 4
    sd = port.make_head_state(E, Q, K, L, 3, ffn=192, seed=7)
    feats = synth.head_inputs(1, E, [(16, 12, 4), (8, 6, 2), (4, 3, 1), (2, 2, 1)], seed=9)
    cl, ml = port.head_forward(feats, sd, E // 32, L, 3)
    assert rel_err(torch.stack(cl), torch.from_numpy(gd["cls"])) < 2e-5
    assert rel_err(ml[-1], torch.from_numpy(gd["mask_last"])) < 2e-5
    assert rel_err(ml[0], torch.from_numpy(gd["mask_first"])) < 2e-5
    pc = [-51.2, -51.2, -5.0, 51.2, 51.2, 3.0]
    res = port.head_simple_test(feats, sd, E // 32, L, [32, 24, 8], 3, points=[synth.lidar_points(50, pc, seed=11)],
                                pc_range=pc)
    assert rel_err(res["output_voxels"][0], torch.from_numpy(gd["output_voxels"])) < 2e-5
    assert rel_err(res["output_points"], torch.from_numpy(gd["output_points"])) < 2e-5


def test_oracle_index_truncation_edge_cases():
    """SURVEY Appendix D.1: values in (-1, 0) truncate to 0 (kept), the upper bound is exclusive."""
    dx, bx, nx = port.gen_dx_bx([-20.0, 20.0, 0.8], [-20.0, 20.0, 0.8], [-2.0, 4.4, 0.8])
    g = torch.tensor([[-20.5, 0.0, 0.0], [-20.9, 0.0, 0.0], [19.99, 0.0, 0.0], [20.0, 0.0, 0.0], [0.0, 0.0, 4.39]])
    idx = port.voxel_index(g, dx, bx)
    assert idx[0, 0] == 0 and idx[1, 0] == -1 and idx[2, 0] == 49 and idx[3, 0] == 50
    gf = torch.cat((idx, torch.zeros(5, 1, dtype=torch.long)), 1)
    assert port.kept_mask(gf, nx).tolist() == [True, False, True, False, True]


def test_oracle_bev_pool_empty_and_duplicates():
    feats = torch.tensor([[1.0, 2.0], [3.0, 4.0], [5.0, 6.0]])
    coords = torch.tensor([[1, 0, 0, 0], [1, 0, 0, 0], [0, 1, 1, 1]])
    out = port.bev_pool(feats, coords, 2, 2, 2, 2)  # (B,C,D=z,H=x,W=y)
    assert out.shape == (2, 2, 2, 2, 2)
    assert out[0, :, 0, 1, 0].tolist() == [4.0, 6.0] and out[1, :, 1, 0, 1].tolist() == [5.0, 6.0]
    assert float(out.sum()) == 21.0
    assert float(port.bev_pool(torch.zeros(0, 2), torch.zeros(0, 4, dtype=torch.long), 1, 1, 1, 1).abs().sum()) == 0


# ------------------------------------------------------------------ drop-in boundary
def test_state_dict_keys_match_reference_contract():
    """our modules carry exactly the reference's state_dict keys/shapes (SURVEY Appendix B; the key lists in
    port.make_*_state were validated by strict load into the REAL reference modules in oracle/validate_port.py)."""
    from occformer_b200.encoder import DualpathTransformerBlock, OccupancyEncoder
    for cin, c, stride in [(128, 128, 1), (128, 256, 2)]:
        sd = port.make_block_state(cin, c, stride, torch.Generator().manual_seed(0))
        blk = DualpathTransformerBlock(cin, c, stride=stride, norm_cfg=dict(type="GN", num_groups=32), layer_index=0)
        mine = blk.state_dict()
        assert set(mine.keys()) == set(sd.keys())
        for k in sd:
            assert tuple(mine[k].shape) == tuple(sd[k].shape), k
        blk.load_state_dict(sd, strict=True)
    enc = OccupancyEncoder(in_channels=128, num_stage=2, block_numbers=[2, 1], block_inplanes=[128, 256],
                           block_strides=[1, 2], out_indices=(0, 1), norm_cfg=dict(type="GN", num_groups=32))
    sd = port.make_encoder_state(128, [128, 256], [2, 1], [1, 2])
    enc.load_state_dict(sd, strict=True)
    assert [b.shift for s in enc.layers for b in s] == [False, True, False]


def test_registry_names():
    from occformer_b200 import BACKBONES, NECKS
    assert BACKBONES.get("OccupancyEncoder") is not None
    assert NECKS.get("ViewTransformerLiftSplatShootVoxel") is not None
    enc = BACKBONES.build(dict(type="OccupancyEncoder", in_channels=128, num_stage=1, block_numbers=[1],
                               block_inplanes=[128], block_strides=[1], out_indices=(0,),
                               norm_cfg=dict(type="GN", num_groups=32, requires_grad=True), with_cp=True))
    assert len(enc.layers) == 1


def test_view_transformer_parameters_match_oracle():
    from occformer_b200.view_transformer import ViewTransformerLiftSplatShootVoxel
    for name, size in (("pr1", (128, 128)), ("nusc_200", (256, 704)), ("nusc_ref", (256, 704))):
        gc = synth.grid_config(name)
        vt = ViewTransformerLiftSplatShootVoxel(grid_config=gc, data_config={"input_size": size}, numC_Trans=128)
        dx, bx, nx = port.gen_dx_bx(gc["xbound"], gc["ybound"], gc["zbound"])
        assert torch.equal(vt.dx.data, dx) and torch.equal(vt.bx.data, bx) and torch.equal(vt.nx.data, nx)
        assert torch.equal(vt.frustum.data, port.create_frustum(size, 16, gc["dbound"]))
        assert vt.D == 112
    with pytest.raises(RuntimeError):  # geometry is a CUDA kernel; CPU tensors are rejected, not computed elsewhere
        vt.get_geometry(**synth.nusc_cameras(1, 6))


def test_product_path_fails_loudly_without_gpu():
    """no CPU fallback: CPU tensors are rejected instead of silently computed elsewhere."""
    from occformer_b200 import ops
    with pytest.raises(RuntimeError):
        ops.gemm(torch.zeros(4, 32), torch.zeros(4, 32))  # CPU tensors
    from occformer_b200.encoder import to_channel_last
    with pytest.raises(RuntimeError):
        to_channel_last(torch.zeros(1, 128, 2, 2, 2))


def test_product_does_not_import_oracle():
    pkg = os.path.join(ROOT, "occformer_b200")
    for dp, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(".py"):
                src = open(os.path.join(dp, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle", src, re.M), f"{f} imports the oracle"
                assert "/root/reference" not in src.replace("under /root/reference", ""), f


# ------------------------------------------------------------------ C ABI
def test_library_binds_every_declaration_with_its_header_types():
    from occformer_b200 import _lib
    assert os.path.exists(_lib.LIB_PATH), "libocc_b200.so not built (python -m occformer_b200.build)"
    l = _lib.lib()  # sets argtypes for every symbol, AttributeError if one is missing
    header = open(os.path.join(ROOT, "include", "occ_b200.h")).read()
    declared = set(re.findall(r"\b(occ_[a-z0-9_]+)\s*\(", header))
    declared -= {"occ_stream_t"}
    assert declared, "no declarations parsed"
    sigs = _lib.signatures()
    assert set(sigs) == declared, "the ctypes binding skipped a declaration"
    for name in declared:
        assert hasattr(l, name), f"{name} declared in include/occ_b200.h but not exported"
        fn = getattr(l, name)
        assert (fn.restype, list(fn.argtypes)) == sigs[name], f"{name}: bound types differ from its declaration"
    assert l.occ_version() >= 100
    # pure host-side helper (no GPU needed)
    assert l.occ_voxel_pool_workspace_bytes(1000, 1, 10, 10, 2) > (200 + 201 + 2000) * 4


def test_header_parser_types(tmp_path):
    """_lib.signatures on the declarations that need more than `int` / pointer: multi-word integer types, a comment
    inside a parameter list, (void); an unknown type or a missing header raises."""
    from ctypes import c_float, c_int, c_longlong, c_size_t, c_uint, c_ulonglong, c_void_p as P
    from occformer_b200 import _lib
    sigs = _lib.signatures()
    assert sigs["occ_version"] == (c_int, [])
    assert sigs["occ_launch_count"] == (c_longlong, [])
    assert sigs["occ_window_layout_rows"] == (c_longlong, [c_int] * 4)
    assert sigs["occ_panoptic_eval_workspace_bytes"] == (c_size_t, [c_longlong])
    assert sigs["occ_panoptic_eval"] == (c_int, [P] * 4 + [c_longlong, c_int, c_uint, c_int, c_int, P, c_size_t, P, P])
    assert sigs["occ_panoptic_voxels"] == (c_int, [P, c_int, P] + [c_int] * 9 + [c_ulonglong, c_int] + [P] * 5 + [P])
    assert sigs["occ_query_head"] == (c_int, [P] * 8 + [c_int] + [P] * 9 + [c_int, P, P, c_float, P, P] + [c_int] * 3 +
                                      [P])
    bad = tmp_path / "bad.h"
    bad.write_text("int occ_ok(const float* x /* (n, C) */, int n);\nshort occ_bad(int a);\n")
    with pytest.raises(RuntimeError, match="occ_bad"):
        _lib.signatures(str(bad))
    with pytest.raises(RuntimeError, match="missing"):
        _lib.signatures(str(tmp_path / "absent.h"))


def test_rejected_call_enqueues_nothing():
    """An argument error returns -1 before any launch: the library's launch count does not move (no GPU needed)."""
    from occformer_b200 import _lib
    l = _lib.lib()
    n0 = l.occ_launch_count()
    assert l.occ_gemm_bf16x3(None, None, None, 1, 1, 32, None, None, 0, 0, None) == -1
    assert l.occ_launch_count() == n0


def test_qkv_head_major_permutation_matches_reference_split():
    """ops.qkv_head_major_perm: the row permutation the encoder applies to WindowMSA.qkv so that a (token, head) reads one
    contiguous [q|k|v] run.  Slicing the permuted projection per head must give the reference's q, k, v of that head
    (window_attention.py:86-88: reshape(B, N, 3, heads, C // heads))."""
    import torch
    from occformer_b200 import ops
    C, heads = 128, 4
    hd = C // heads
    perm = ops.qkv_head_major_perm(C, heads)
    assert sorted(perm.tolist()) == list(range(3 * C))
    g = torch.Generator().manual_seed(0)
    x = torch.randn(5, C, generator=g)
    w, b = torch.randn(3 * C, C, generator=g), torch.randn(3 * C, generator=g)
    ref = torch.nn.functional.linear(x, w, b).view(5, 3, heads, hd)        # [token, q|k|v, head, d]
    hm = torch.nn.functional.linear(x, w[perm], b[perm]).view(5, heads, 3, hd)  # [token, head, q|k|v, d]
    assert torch.equal(hm.permute(0, 2, 1, 3), ref)


def test_neck_port_vs_reference_golden():
    """MSDeformAttnPixelDecoder3D (SURVEY.md 8(f)1, the first "next" row): the oracle restatement reproduces the outputs
    the reference module produced under the shim (tests/golden/neck_small.npz, oracle/gen_golden.py neck).  No CUDA
    implementation of the neck exists yet; this pins its oracle for the next round."""
    from oracle import port
    from util import golden
    c = port.NECK_CASE
    sd = port.make_neck_state(c["in_channels"], c["E"], c["layers"], c["heads"], c["levels"], c["points"], c["ffn"],
                              seed=c["wseed"])
    feats = port.neck_inputs(c, B=1)
    outs = port.ms_deform_pixel_decoder_3d(feats, sd, c["strides"], c["heads"], c["layers"], c["levels"], c["points"])
    gold = golden("neck_small.npz")
    assert len(outs) == 4
    for i, o in enumerate(outs):
        assert_close(o, torch.from_numpy(gold[f"out{i}"]), 2e-5, f"neck port out[{i}] vs reference golden")


# ------------------------------------------------------------------ boundary: DepthNet + the unmodified reference configs
def test_depthnet_vs_reference_golden():
    """occformer_b200.depthnet.DepthNet (SURVEY.md 8(f)3) loads the REFERENCE class's own state_dict strictly and
    reproduces its output (tests/golden/depthnet_small.npz: reference DepthNet under the shim, oracle/gen_golden.py;
    the shim's DCN is an explicit-gather restatement of mmcv's DeformConv2dPack, ours goes through grid_sample)."""
    from oracle.gen_golden import DEPTHNET_CASE as c
    from occformer_b200.depthnet import DepthNet
    gd = golden("depthnet_small.npz")
    sd = {k[2:]: torch.from_numpy(gd[k]) for k in gd.files if k.startswith("w:")}
    net = DepthNet(c["cin"], c["mid"], c["ctx"], c["D"], cam_channels=c["cam"]).eval()
    net.load_state_dict(sd, strict=True)
    g = torch.Generator().manual_seed(c["xseed"])
    x = torch.randn(c["B"] * c["N"], c["cin"], c["fH"], c["fW"], generator=g)
    mlp = torch.randn(c["B"], c["N"], c["cam"], generator=g)
    with torch.no_grad():
        y = net(x, mlp)
    assert_close(y, torch.from_numpy(gd["out"]), 1e-5, "DepthNet vs reference golden")


@pytest.mark.parametrize("name", ["nusc_r50", "kitti"])
def test_modules_build_from_unmodified_reference_config(name):
    """The four hot-path sections of the reference's own config files (tests/golden/model_cfg_*.json = the ``model`` dict
    of projects/configs/occformer_{nusc/occformer_nusc_r50_256x704,kitti/occformer_kitti}.py, extracted verbatim by
    oracle/gen_golden.py) build through our registries, with the reference's state_dict key sets."""
    import json
    from occformer_b200 import BACKBONES, HEADS, NECKS, POSITIONAL_ENCODING
    cfg = json.load(open(os.path.join(GOLDEN, f"model_cfg_{name}.json")))
    vt = NECKS.build(cfg["img_view_transformer"])
    enc = BACKBONES.build(cfg["img_bev_encoder_backbone"])
    neck = NECKS.build(cfg["img_bev_encoder_neck"])
    head = HEADS.build(cfg["pts_bbox_head"])
    assert POSITIONAL_ENCODING.get("SinePositionalEncoding3D") is not None
    kitti = name == "kitti"
    assert vt.D == 112 and vt.cam_channels == (33 if kitti else 27) and vt.numC_input == (640 if kitti else 512)
    assert vt.grid_size() == (128, 128, 16)
    assert len(enc.layers) == 4 and [len(l) for l in enc.layers] == [2, 2, 2, 2]
    assert neck.num_encoder_levels == 3 and len(neck.encoder.layers) == 6 and neck.num_heads == 8
    assert head.num_queries == 100 and head.num_classes == (20 if kitti else 17) and head.num_transformer_decoder_layers == 9
    # state_dict contracts: encoder / neck / head keys == the key sets validated against the real reference classes
    E = 192
    assert set(enc.state_dict()) == set(synth.make_encoder_state(128, [128, 256, 512, 1024], [2, 2, 2, 2], [1, 2, 2, 2]))
    assert set(neck.state_dict()) == set(synth.make_neck_state([128, 256, 512, 1024], E, 6, 8, 3, 4, 4 * E))
    assert set(head.state_dict()) == set(synth.make_head_state(E, 100, 20 if kitti else 17, 9, 3))
    if not kitti:  # img_view_transformer.* of a reference checkpoint: dx / bx / nx / frustum + depth_net.*
        want = json.load(open(os.path.join(GOLDEN, "depthnet_keys_nusc.json")))
        mine = {k[len("depth_net."):]: list(v.shape) for k, v in vt.state_dict().items() if k.startswith("depth_net.")}
        assert mine == want, "depth_net.* keys / shapes differ from the reference DepthNet(512, 512, 128, 112, cam_channels=27)"
        assert {k for k in vt.state_dict() if not k.startswith("depth_net.")} == {"dx", "bx", "nx", "frustum"}
    # get_mlp_input (occupancyformer.py:77) matches cam_channels
    B, N = 1, (1 if kitti else 6)
    r, t = torch.eye(3).view(1, 1, 3, 3).repeat(B, N, 1, 1), torch.zeros(B, N, 3)
    k = torch.eye(4).view(1, 1, 4, 4).repeat(B, N, 1, 1) if kitti else r
    bda = torch.eye(4).view(1, 4, 4) if kitti else torch.eye(3).view(1, 3, 3)
    assert vt.get_mlp_input(r, t, k, r, t, bda).shape == (B, N, vt.cam_channels)


# ------------------------------------------------------------------ A18 / A19: class-guided sampling (host functions, RNG driven)
def test_class_guided_sampling_host_functions():
    """Distributional / structural checks only (SURVEY.md 8(a): RNG driven, not parity-checkable bit-wise)."""
    from occformer_b200 import sampling as S
    torch.manual_seed(0)
    shape = (12, 10, 6)
    idx = torch.randint(0, 720, (3, 50))
    assert np.array_equal(S.unravel_indices(idx, shape).numpy(), np.stack(np.unravel_index(idx.numpy(), shape), -1))
    vol = torch.randn(2, 1, *shape)
    pts = torch.rand(2, 40, 3)
    got = S.point_sample_3d(vol, pts[..., [2, 1, 0]], align_corners=True)
    ref = torch.nn.functional.grid_sample(vol, (pts[..., [2, 1, 0]] * 2 - 1)[:, :, None, None], align_corners=True)[..., 0, 0]
    assert torch.equal(got, ref) and got.shape == (2, 1, 40)
    # two instances: a rare class (label 2, high weight) and a frequent one (label 1); voxels outside both are never drawn
    gt_labels = torch.tensor([1, 2])
    gt_masks = torch.zeros(2, *shape)
    gt_masks[0, :6] = 1
    gt_masks[1, 8:] = 1
    w = S.class_sampling_weights(S.SEMANTIC_KITTI_CLASS_FREQUENCIES, 0.25)
    assert w.min() == 1.0 and w[2] > w[1] > w[0]
    pidx, pc = S.sample_valid_coords_with_frequencies(300, gt_labels, gt_masks, sample_weights=w)
    occ = (gt_masks.sum(0) > 0).view(-1)
    assert bool(occ[pidx].all()) and pidx.unique().numel() == 300 and float(pc.min()) >= 0 and float(pc.max()) <= 1
    frac_rare = float((gt_masks[1].view(-1)[pidx] > 0).float().mean())
    assert frac_rare > 0.5, "the rare class (3.4x the weight, 2/5 of the valid voxels) must dominate the draw"
    mask_pred = torch.randn(2, *shape)
    bi, bc = S.get_uncertain_point_coords_3d_with_frequency(mask_pred, None, [gt_labels], [gt_masks], w, 64, 3.0, 0.75)
    assert bi.shape == (2, 64) and bc.shape == (2, 64, 3) and bool(occ[bi].all())
    # the importance-sampled part are the most uncertain of the over-sampled candidates: |logit| there is small on average
    assert float(mask_pred.view(2, -1).gather(1, bi[:, :48]).abs().mean()) < float(mask_pred.abs().mean())
    lidar = [torch.cat([torch.rand(30, 3) * 20 - 10, torch.ones(30, 1)], 1)]
    c = S.get_nusc_lidarseg_point_coords(torch.randn(2, 1, *shape), lidar, [gt_labels], 40, 3.0, 0.75, [-10, -10, -10, 10, 10, 10])
    assert c.shape == (2, 40, 3)


def test_window_layout_index_matches_window_token_row():
    """ops.window_layout_index (token row -> row of the window-layout buffer the fused attention kernel loads by TMA) is the
    inverse of the window -> token map of ShiftWindowMSA (window_attention.py:168-242: pad, roll by -3, 7x7 partition),
    restated here window by window."""
    import torch
    from occformer_b200 import ops

    def brute(B, X, Y, Z, shift):
        nWx, nWy = (X + 6) // 7, (Y + 6) // 7
        Xp, Yp = nWx * 7, nWy * 7
        out = torch.full((B * X * Y * (Z + 1),), -1, dtype=torch.long)
        for img in range(B * (Z + 1)):
            for wx in range(nWx):
                for wy in range(nWy):
                    for t in range(49):
                        i, j = divmod(t, 7)
                        x, y = wx * 7 + i, wy * 7 + j
                        if shift:
                            x, y = (x + 3) % Xp, (y + 3) % Yp
                        if x >= X or y >= Y:
                            continue
                        if img < B * Z:
                            b, z = divmod(img, Z)
                            r = ((b * X + x) * Y + y) * Z + z
                        else:
                            r = B * X * Y * Z + ((img - B * Z) * X + x) * Y + y
                        out[r] = ((wx * nWy + wy) * (B * (Z + 1)) + img) * 64 + t
        return out

    for cfg in [(1, 14, 7, 1, False), (1, 10, 16, 2, True), (2, 15, 10, 4, False), (1, 33, 40, 3, True)]:
        got = ops.window_layout_index(*cfg)
        assert torch.equal(got, brute(*cfg)), cfg
        assert got.unique().numel() == got.numel()


def test_host_helpers_pad_head_rows():
    """host-side operand helper of the neck: per-head padding of value_proj (128-byte head slices)"""
    import torch
    from occformer_b200 import ops
    g = torch.Generator().manual_seed(0)
    E, H = 192, 8
    w, b = torch.randn(E, E, generator=g), torch.randn(E, generator=g)
    wp, bp = ops.pad_head_rows(w, b, H)
    assert wp.shape == (H * 32, E) and bp.shape == (H * 32,)
    x = torch.randn(5, E, generator=g)
    y, yp = x @ w.t() + b, (x @ wp.t() + bp).view(5, H, 32)
    assert torch.allclose(yp[:, :, :24].reshape(5, E), y, atol=1e-5) and float(yp[:, :, 24:].abs().max()) == 0.0
    w32, b32 = ops.pad_head_rows(torch.randn(256, 64, generator=g), torch.randn(256, generator=g), 8)  # hd = 32: unchanged
    assert w32.shape == (256, 64)
