"""The view transformer built from a model config, and its pooled output against the oracle chain (oracle.port lift and
voxel pooling): shared by the GPU tests that run DepthNet, ResNet-50 + SECONDFPN or EfficientNet-B7 into it."""
import json
import os

import torch

from util import GOLDEN, assert_close, parity_log, rel_err
from occformer_b200 import NECKS, ops, synth


def config_view_transformer(case, seed, B):
    """The view transformer of tests/golden/model_cfg_<case>.json (eval mode, on the host) with the synthetic DepthNet
    state of `seed`, whose mlp_input BatchNorm1d running statistics match the case's B cameras (as a trained model's
    would).  -> (vt, cams, mlp_input)"""
    vt = NECKS.build(json.load(open(os.path.join(GOLDEN, f"model_cfg_{case}.json")))["img_view_transformer"])
    dn = vt.depth_net
    sd = synth.make_depthnet_state(dn.in_channels, dn.mid_channels, dn.context_channels, dn.depth_channels,
                                   dn.cam_channels, seed=seed)
    cams = synth.workload_cameras("kitti" if case == "kitti" else "nusc_ref", B)
    mlp = vt.get_mlp_input(cams["rots"], cams["trans"], cams["intrins"], cams["post_rots"], cams["post_trans"],
                           cams["bda"])
    sd["bn.running_mean"] = mlp.reshape(-1, dn.cam_channels).mean(0)
    sd["bn.running_var"] = mlp.reshape(-1, dn.cam_channels).var(0, unbiased=False) + 1.0
    dn.load_state_dict(sd, strict=True)
    return vt.eval(), cams, mlp


def check_pooled(vt, cams, depth_out64, prob, bev, B, N, what, grid_gate):
    """vt's depth_prob and pooled grid bev against oracle.port's lift of depth_out64 (DepthNet's output in float64) and
    its pooling over the kernel's own voxel assignment.  The kernel recomputes the geometry in fp32, so a point may
    change voxel only within 1e-4 cells of a cell boundary; pooled over the kernel's assignment, such a point does not
    decide the comparison.  grid_gate "exact": assert_close on the grid; "terms": every voxel within 1e-2 of the
    magnitude of its terms and the grid within 1e-3 of its largest value (a chain from images)."""
    from oracle import port
    D, ctx = vt.D, vt.numC_Trans
    vol, want_prob = port.lift(depth_out64[:, :D], depth_out64[:, D:D + ctx], B, N)
    gc = vt.grid_config
    frustum = port.create_frustum(vt.data_config["input_size"], vt.downsample, gc["dbound"])
    geom = port.get_geometry(frustum, **cams)
    dx, bx, nx = port.gen_dx_bx(gc["xbound"], gc["ybound"], gc["zbound"])
    _, gf, kept = port.voxel_pooling(geom, vol[..., :1], dx, bx, nx)
    X, Y, Z = vt.grid_size()
    vox = ops._workspace(gf.shape[0], B, X, Y, Z, bev.device).vox_id.cpu().long()
    ref_lin = ((gf[:, 3] * X + gf[:, 0]) * Y + gf[:, 1]) * Z + gf[:, 2]
    flips = vox != torch.where(kept, ref_lin, torch.full_like(ref_lin, -1))
    frac = (geom.view(-1, 3) - (bx - dx / 2.0)) / dx
    assert bool((~flips | ((frac - frac.round()).abs() < 1e-4).any(-1)).all()), "index flips away from cell boundaries"
    rows, keep = vol.reshape(-1, ctx), vox >= 0
    want = torch.zeros(B * X * Y * Z, ctx, dtype=torch.float64).index_add_(0, vox[keep], rows[keep])
    rp = assert_close(prob, want_prob, 1e-3, f"{what} depth_prob")
    line = f"{what}: depth_prob rel_max {rp:.2e}, "
    if grid_gate == "exact":
        rg = assert_close(bev, want.view(B, X, Y, Z, ctx).permute(0, 4, 1, 2, 3), 1e-3, f"{what} pooled grid")
        line += f"grid rel_max {rg:.2e}"
    else:
        # A voxel is a sum of up to hundreds of signed point terms prob * feature, so its error scales with the sum of
        # their magnitudes, not with its value (a few voxels cancel to near zero); and a softmax probability carries the
        # absolute error of its logit as a relative one (1e-4 of logits of magnitude tens).  The magnitude's floor of
        # 1e-3 of the grid's largest value covers points of a vanishing depth probability (fp32 denormals).
        assert grid_gate == "terms", grid_gate
        got = bev.permute(0, 2, 3, 4, 1).reshape(-1, ctx).double().cpu()
        scale = torch.zeros(B * X * Y * Z, ctx, dtype=torch.float64).index_add_(0, vox[keep], rows[keep].abs())
        scale = scale + 1e-3 * float(want.abs().max())
        worst = float(((got - want).abs() / scale).max())
        assert worst <= 1e-2, f"{what}: a voxel off by {worst:.2e} of the magnitude of its terms"
        rg = rel_err(got, want)
        assert rg <= 1e-3, f"{what}: pooled grid rel_max {rg:.2e}"
        line += f"grid rel_max {rg:.2e}, worst voxel {worst:.2e} of its terms' magnitude"
    parity_log(f"{line}, {int(flips.sum())} boundary flips of {flips.numel()} points")
