"""The OccupancyFormer detector on the H100: the unmodified configs' ``model`` dicts (tests/golden/detector_cfg_*.json),
built through DETECTORS, with the synthetic weights of synth.make_detector_state loaded by one
``load_state_dict(strict=True)``, run from normalised camera images to the reference test loop's outputs.

1. images -> outputs against the oracle at the configs' real sizes (nuScenes R50: 6 x 256x704, KITTI B7: 384x1280,
   nuScenes R101-DCN: 6 x 896x1600): the image encoder and DepthNet in float64 (their torch restatements; on the GPU for
   R101, as tests/test_gpu_resnet_dcn.py runs them, on the host otherwise), then oracle.port on the host for lift,
   pooling, encoder, pixel decoder and head, as tests/test_gpu_fullsize.py chains them.
2. simple_test is the module chain called by hand in the reference's order (batch 2).
3. a batch of 2 equals two batch-1 calls (the (B, N) <-> B*N views).
4. model(return_loss=False, ...) as the reference's test loop calls it: keys, dtypes, shapes, evaluation_semantic.
5. the panoptic config: the head's ids, with target_* attached.
6. CUDA graph, launch count and kernel names (tests/detector_trace.py, in a process of its own).

Repeat runs: the pooling kernel sums a voxel's points in the order its atomics pushed them onto the voxel's list, so
two calls can differ in the last bits of the pooled grid, and everything after it by the error of that reordering.
Everything before the pooling is compared bit for bit; the pooled grid has the same non-empty voxels and sums equal to
fp32 summation-order accuracy; the outputs are bit for bit when the sums came out identical and otherwise within the
1e-3 gate with label agreement > 0.9999 (the decoder's attention-mask threshold is discontinuous, tests/test_gpu_fullsize.py).
"""
import json
import os

import numpy as np
import pytest
import torch

from util import GOLDEN, assert_close, f64, images, parity_log, run_script
from vt_chain import check_pooled
from occformer_b200 import DETECTORS, synth

pytestmark = pytest.mark.gpu

# the workload whose output grid, point-cloud range and classes a config has, and the one whose cameras it sees
WL = {"nusc_r50": "nusc_ref", "nusc_r101": "nusc_ref", "nusc_panoptic": "nusc_panoptic", "kitti": "kitti"}
CAMS = {"nusc_r50": "nusc_ref", "nusc_r101": "nusc_r101", "nusc_panoptic": "nusc_ref", "kitti": "kitti"}


def _cfg(name):
    return json.load(open(os.path.join(GOLDEN, f"detector_cfg_{name}.json")))


def _cams(name, B):
    return synth.workload_cameras(CAMS[name], B)


def detector(name, dev, seed=0):
    """-> (model on dev in eval mode, its state_dict on the host)"""
    cfg = _cfg(name)
    model = DETECTORS.build(cfg).eval()
    sd = synth.make_detector_state(cfg, seed=seed, cams=_cams(name, 1))
    model.load_state_dict(sd, strict=True)
    return model.to(dev), sd


def inputs(name, B, dev, seed=1, npts=0):
    """the reference loader's test-time sample: img_metas, img_inputs = [imgs, rots, trans, intrins, post_rots,
    post_trans, bda, gt_depths, sensor2sensors], gt_occ and (npts > 0) points_occ (x, y, z, label)"""
    wl = synth.WORKLOADS[WL[name]]
    N, (H, W) = synth.WORKLOADS[CAMS[name]]["cams"], synth.WORKLOADS[CAMS[name]]["input_size"]
    cams = _cams(name, B)
    imgs = images(B * N, H, W, seed=seed).view(B, N, 3, H, W)
    img_inputs = [imgs] + [cams[k] for k in ("rots", "trans", "intrins", "post_rots", "post_trans", "bda")]
    img_inputs += [torch.zeros(B, N, H, W), torch.eye(4).expand(B, N, 4, 4).contiguous()]
    metas = [dict(occ_size=list(wl["occ"]), pc_range=list(wl["pc"])) for _ in range(B)]
    g = torch.Generator().manual_seed(seed + 1)
    gt_occ = torch.randint(0, wl["classes"], (B, *wl["occ"]), generator=g)
    pts = None
    if npts:
        pts = []
        for b in range(B):
            p = synth.lidar_points(npts, wl["pc"], seed=seed + 2 + b)[:, :3]
            pts.append(torch.cat([p, torch.randint(0, 17, (npts, 1), generator=g).float()], dim=1).to(dev))
    return metas, [t.to(dev) for t in img_inputs], gt_occ.to(dev), pts


class Taps:
    """forward hooks on the detector's submodules: each one's last output, copied to the host"""

    def __init__(self, model):
        def keep(name):
            def hook(mod, args, out):
                self.out[name] = _host(out)
            return hook
        self.out = {}
        self.handles = [getattr(model, n).register_forward_hook(keep(n)) for n in
                        ("img_neck", "img_view_transformer", "img_bev_encoder_backbone", "img_bev_encoder_neck")]

    def close(self):
        for h in self.handles:
            h.remove()


def _host(out):
    if isinstance(out, (list, tuple)):
        return type(out)(_host(o) for o in out)
    return out.detach().float().cpu().clone() if torch.is_tensor(out) else out


def _bits_equal(a, b):
    a, b = a.detach().cpu().contiguous(), b.detach().cpu().contiguous()
    return a.shape == b.shape and torch.equal(a.view(torch.int32) if a.dtype == torch.float32 else a,
                                              b.view(torch.int32) if b.dtype == torch.float32 else b)


def same_run(a, b, what):
    """two runs of the pooled path: bit for bit, or within the gate (module docstring)"""
    if _bits_equal(a["output_voxels"], b["output_voxels"]):
        assert torch.equal(a["output_labels"].cpu(), b["output_labels"].cpu()), what
        parity_log(f"[detector] {what}: bit for bit")
        return
    assert_close(a["output_voxels"], b["output_voxels"], what=f"{what} output_voxels")
    agree = float((a["output_labels"].cpu() == b["output_labels"].cpu()).double().mean())
    parity_log(f"[detector] {what}: within the gate (pooled sums reordered), label agreement {100 * agree:.4f} %")
    assert agree > 0.9999, what


def same_grid(a, b, what):
    assert torch.equal(a.abs().sum(1) != 0, b.abs().sum(1) != 0), f"{what}: non-empty voxels differ"
    assert_close(a, b, 1e-5, f"{what} pooled grid")


# ------------------------------------------------------------------ 1. images -> outputs vs the host oracle
def _oracle(name, model, sd, img_inputs, metas, cams, dev):
    """the oracle chain of one sample: the float64 torch forwards of image encoder + DepthNet on `dev`, then oracle.port
    (fp32) on the host from lift to head"""
    from oracle import port
    vt, cfg_neck, head = model.img_view_transformer, model.img_bev_encoder_neck, model.pts_bbox_head
    imgs = img_inputs[0].double().to(dev)
    B, N = imgs.shape[:2]
    with torch.no_grad():
        stages = f64(model.img_backbone, dev)._forward_torch(imgs.flatten(0, 1))
        feat = f64(model.img_neck, dev)._forward_torch(list(stages))[0]
        del stages
        mlp = vt.get_mlp_input(*[t.cpu() for t in img_inputs[1:7]])
        depth = f64(vt.depth_net, dev)._forward_torch(feat, mlp.double().to(dev)).cpu()
        feat = feat.cpu()
    D, C = vt.D, vt.numC_Trans
    gc = vt.grid_config
    frustum = port.create_frustum(vt.data_config["input_size"], vt.downsample, gc["dbound"])
    geom = port.get_geometry(frustum, **cams)
    vol, _ = port.lift(depth[:, :D].float(), depth[:, D:D + C].float(), B, N)
    dx, bx, nx = port.gen_dx_bx(gc["xbound"], gc["ybound"], gc["zbound"])
    grid, _, _ = port.voxel_pooling(geom, vol, dx, bx, nx)
    del vol

    def sub(prefix):
        return {k[len(prefix):]: v for k, v in sd.items() if k.startswith(prefix)}
    e = _cfg(name)["img_bev_encoder_backbone"]
    enc = port.occupancy_encoder(grid, sub("img_bev_encoder_backbone."), e["block_numbers"], e["block_strides"],
                                 tuple(e["out_indices"]))
    n = cfg_neck
    feats = port.ms_deform_pixel_decoder_3d(enc, sub("img_bev_encoder_neck."), n.strides, n.num_heads,
                                            len(n.encoder.layers), n.num_encoder_levels, n.num_points)
    res = port.head_simple_test(feats, sub("pts_bbox_head."), head.num_heads, head.num_transformer_decoder_layers,
                                metas[0]["occ_size"], head.num_transformer_feat_level)
    return dict(feat=feat, depth=depth, enc=enc, feats=feats, vox=res["output_voxels"][0])


@pytest.mark.parametrize("name", ["nusc_r50", "kitti", "nusc_r101"])
def test_images_to_outputs_vs_oracle(cuda, name):
    torch.set_num_threads(min(os.cpu_count() or 1, 32))
    model, sd = detector(name, cuda, seed=10)
    metas, img_inputs, gt_occ, _ = inputs(name, 1, cuda, seed=11)
    taps = Taps(model)
    out = model.simple_test(metas, img_inputs, gt_occ=gt_occ)
    torch.cuda.synchronize()
    taps.close()
    got = taps.out
    cams = {k: t.cpu() for k, t in zip(("rots", "trans", "intrins", "post_rots", "post_trans", "bda"), img_inputs[1:7])}
    # R101-DCN in float64 on the host would take many minutes; its torch forward runs on the device instead
    ref = _oracle(name, model, sd, img_inputs, metas, cams, cuda if name == "nusc_r101" else torch.device("cpu"))
    tag = f"[detector {name}]"
    failed = []

    def gate(a, b, what):  # every stage is reported before the test fails
        try:
            assert_close(a, b, what=what)
        except AssertionError as e:
            failed.append(str(e))

    gate(got["img_neck"][0], ref["feat"], f"{tag} image features")
    bev, prob = got["img_view_transformer"]
    N = img_inputs[0].shape[1]
    # (on the device: check_pooled reads the kernel's voxel assignment from the pooling workspace of that device)
    check_pooled(model.img_view_transformer, cams, ref["depth"], prob, bev.to(cuda), 1, N,
                 f"{tag} images -> view transformer", "terms")
    for i, (o, r) in enumerate(zip(got["img_bev_encoder_backbone"], ref["enc"])):
        gate(o, r, f"{tag} encoder out[{i}] {tuple(r.shape)}")
    for i, (o, r) in enumerate(zip(got["img_bev_encoder_neck"], ref["feats"])):
        gate(o, r, f"{tag} pixel decoder out[{i}] {tuple(r.shape)}")
    gate(out["output_voxels"], ref["vox"], f"{tag} output_voxels {tuple(ref['vox'].shape)}")
    agree = float((out["output_labels"].long().cpu() == ref["vox"].argmax(1)).double().mean())
    parity_log(f"[parity] {tag} images -> outputs label agreement {100 * agree:.4f} %")
    assert not failed, "\n".join(failed)
    assert agree > 0.9999


# ------------------------------------------------------------------ 2. the detector is the module chain
def test_simple_test_is_the_module_chain(cuda):
    model, _ = detector("nusc_r50", cuda, seed=20)
    metas, img_inputs, gt_occ, _ = inputs("nusc_r50", 2, cuda, seed=21)
    taps = Taps(model)
    out = model.simple_test(metas, img_inputs, gt_occ=gt_occ)
    taps.close()
    with torch.no_grad():
        imgs = img_inputs[0]
        B, N, C, H, W = imgs.shape
        x = model.img_neck(model.img_backbone(imgs.view(B * N, C, H, W)))[0]
        x = x.view(B, N, *x.shape[1:])
        vt = model.img_view_transformer
        mlp = vt.get_mlp_input(*img_inputs[1:7])
        bev, prob = vt([x] + list(img_inputs[1:7]) + [mlp])
        enc = model.img_bev_encoder_backbone(bev)
        feats = model.img_bev_encoder_neck(enc)
        want = model.pts_bbox_head.simple_test(feats, metas)
    assert _bits_equal(taps.out["img_neck"][0], x.view(B * N, *x.shape[2:])), "image features"
    assert _bits_equal(taps.out["img_view_transformer"][1], prob), "depth_prob"
    same_grid(taps.out["img_view_transformer"][0], bev.cpu(), "[detector vs chain]")
    same_run(out, dict(want, output_voxels=want["output_voxels"][0]), "detector vs the modules by hand")
    assert out["target_voxels"] is gt_occ and out["output_points"] is None


# ------------------------------------------------------------------ 3. samples are independent
def test_batch_of_two_is_two_batches_of_one(cuda):
    model, _ = detector("nusc_r50", cuda, seed=30)
    metas, img_inputs, gt_occ, _ = inputs("nusc_r50", 2, cuda, seed=31)
    taps = Taps(model)
    both = model.simple_test(metas, img_inputs, gt_occ=gt_occ)
    t2 = dict(taps.out)
    for b in range(2):
        one = model.simple_test(metas[b:b + 1], [t[b:b + 1] for t in img_inputs], gt_occ=gt_occ[b:b + 1])
        N = img_inputs[0].shape[1]
        assert _bits_equal(taps.out["img_neck"][0], t2["img_neck"][0][b * N:(b + 1) * N]), f"sample {b} image features"
        assert _bits_equal(taps.out["img_view_transformer"][1], t2["img_view_transformer"][1][b * N:(b + 1) * N]), \
            f"sample {b} depth_prob"
        same_grid(taps.out["img_view_transformer"][0], t2["img_view_transformer"][0][b:b + 1], f"[sample {b}]")
        same_run(one, {k: both[k][b:b + 1] for k in ("output_voxels", "output_labels")}, f"sample {b} of a batch of 2")
    taps.close()


# ------------------------------------------------------------------ 4. the reference test loop's call
def test_reference_test_loop_call(cuda):
    model, _ = detector("nusc_r50", cuda, seed=40)
    metas, img_inputs, gt_occ, pts = inputs("nusc_r50", 1, cuda, seed=41, npts=3000)
    res = model(return_loss=False, rescale=True, img_metas=metas, img_inputs=img_inputs, gt_occ=gt_occ, points_occ=pts)
    assert set(res) == {"output_voxels", "output_points", "output_labels", "evaluation_semantic", "target_points",
                        "target_voxels"}
    assert res["output_voxels"].shape == (1, 17, 256, 256, 32) and res["output_voxels"].dtype == torch.float32
    assert res["output_points"].shape == (3000,) and res["output_points"].dtype == torch.int64
    assert int(res["output_points"].min()) >= 1 and int(res["output_points"].max()) <= 16
    assert res["target_voxels"] is gt_occ
    assert torch.equal(res["target_points"], torch.cat(pts))
    ev = res["evaluation_semantic"]
    assert type(ev) is np.ndarray and ev.dtype == np.int64 and ev.shape == (16, 16)
    # fast_hist_crop(output_points, target_points[:, 3], np.arange(16)) on the host (metric_util.py:8-23)
    pred, gt = res["output_points"].cpu().numpy(), res["target_points"][:, 3].cpu().numpy().astype(int)
    n = 17
    k = (gt >= 0) & (gt < n)
    hist = np.bincount(n * gt[k] + pred[k], minlength=n * n)[:n * n].reshape(n, n)[1:, 1:]
    assert np.array_equal(ev, hist) and ev.sum() > 0
    # the labels are the argmax of the head's point scores
    scores = model.pts_bbox_head.simple_test(model.extract_feat(None, img_inputs, metas)[0], metas, points=pts)
    agree = float((torch.argmax(scores["output_points"][:, 1:], 1) + 1 == res["output_points"]).double().mean())
    assert agree > 0.999


# ------------------------------------------------------------------ 5. panoptic head: the head's dict, target_* attached
def test_panoptic_config(cuda):
    model, _ = detector("nusc_panoptic", cuda, seed=50)
    metas, img_inputs, gt_occ, pts = inputs("nusc_panoptic", 1, cuda, seed=51, npts=2000)
    taps = Taps(model)
    res = model(return_loss=False, rescale=True, img_metas=metas, img_inputs=img_inputs, gt_occ=gt_occ, points_occ=pts)
    taps.close()
    feats = [f.to(cuda) for f in taps.out["img_bev_encoder_neck"]]
    want = model.pts_bbox_head.simple_test(feats, metas, points=pts)
    assert set(res) == set(want) | {"target_voxels", "target_points"}
    assert res["target_voxels"] is gt_occ and torch.equal(res["target_points"], torch.cat(pts))
    sem, pan = res["output_voxels"][0]
    assert sem.dtype == torch.int64 and sem.shape == (1, 256, 256, 32)
    for got, ref, what in ((sem, want["output_voxels"][0][0], "semantic"), (pan, want["output_voxels"][0][1], "panoptic"),
                           (res["output_points"], want["output_points"], "point labels"),
                           (res["output_panoptic_points"], want["output_panoptic_points"], "point panoptic ids")):
        agree = float((got == ref).double().mean())
        parity_log(f"[detector panoptic] {what}: {100 * agree:.4f} % equal to head.simple_test on the tapped features")
        assert agree > 0.9999, what


# ------------------------------------------------------------------ 6. one graph, only library work
def test_cuda_graph_launch_count_and_kernels(cuda):
    res = run_script("detector_trace.py", timeout=1200)
    print(res)
    assert res["counted"] == res["kernels"] + res["memsets"], "the launch counter and the trace disagree"
    assert res["counted"] == sum(res["per_module"].values()), res["per_module"]
    assert not res["unexpected"], f"GPU work that is neither the library's nor a listed small torch op: {res['unexpected']}"
    assert not any("cudnn" in n.lower() or "cublas" in n.lower() or "gemm" in n.lower() for n in res["other"])
    assert res["other_ms"] < 1e-3 * res["total_ms"], f"torch kernels take {res['other_ms']} of {res['total_ms']} ms"
    assert res["graph_equals_eager"] or res["graph_within_gate"], "CUDA-graph replay differs from the eager call"
