"""SemanticKITTI ground truth from the voxel files on the H100 (targets.semantic_kitti_occupancy, csrc/semkitti_labels.cu),
bit for bit: against the reference's preprocessing (tests/golden/semkitti_labels.npz) and against the numpy restatement
(oracle/semkitti_labels.py, itself checked against the reference) on full-size synthetic frames; then the detector's
simple_test with the voxel files in its metas."""
import os

import numpy as np
import pytest
import torch

from util import GOLDEN, graph_replay
from oracle import semkitti_labels as sk
from occformer_b200 import ops, targets

pytestmark = pytest.mark.gpu

MODES = ("mixed", "no_invalid", "all_invalid", "sparse", "structured")


@pytest.fixture(scope="module")
def gold():
    return dict(np.load(os.path.join(GOLDEN, "semkitti_labels.npz")))


@pytest.fixture(scope="module")
def lm(gold):
    return {int(k): int(v) for k, v in gold["learning_map"]}


def test_fixture_frames_equal_reference(cuda, gold, lm):
    labels = [gold[f"{m}_label"].tobytes() for m in sk.MODES]
    invalids = [gold[f"{m}_invalid"].tobytes() for m in sk.MODES]
    out = targets.semantic_kitti_occupancy(labels, invalids, lm)
    assert out.shape == (len(sk.MODES), 256, 256, 32) and out.dtype == torch.int64 and out.device == cuda
    for b, m in enumerate(sk.MODES):
        assert torch.equal(out[b].cpu(), torch.from_numpy(gold[f"{m}_gt"].astype(np.int64))), m
    one = targets.semantic_kitti_occupancy(labels[0], invalids[0], lm)  # one sample: (256, 256, 32)
    assert torch.equal(one, out[0])


def test_every_mode_equals_restatement_batch4(cuda, lm):
    frames = [sk.synthetic_voxels(lm, 100 + i, m) for i, m in enumerate(MODES)]
    ref = [sk.occupancy(lab, inv, lm) for lab, inv in frames]
    # every learning-map key and every unknown key below the LUT size is in the mixed frame
    lab0 = np.frombuffer(frames[0][0], np.uint16)
    assert set(lm) <= set(lab0.tolist()) and set(range(max(lm) + 1, max(lm) + 100)) <= set(lab0.tolist())
    assert (ref[2] == 255).all() and not (ref[1] == 255).all()
    for sl in (slice(0, 4), slice(1, 5)):
        out = targets.semantic_kitti_occupancy([f[0] for f in frames[sl]], [f[1] for f in frames[sl]], lm).cpu()
        for b, r in enumerate(ref[sl]):
            n_bad = int((out[b].numpy() != r).sum())
            assert n_bad == 0, f"{MODES[sl][b]}: {n_bad} voxels differ"


def test_numpy_and_bytearray_inputs(cuda, lm):
    lab, inv = sk.synthetic_voxels(lm, 5, "mixed")
    a = targets.semantic_kitti_occupancy([np.frombuffer(lab, np.uint16)], [bytearray(inv)], lm)
    assert torch.equal(a[0].cpu(), torch.from_numpy(sk.occupancy(lab, inv, lm)))


@pytest.mark.parametrize("value", [359, 360, 65535])
def test_label_past_the_lut_raises(cuda, lm, value):
    lab, inv = sk.synthetic_voxels(lm, 6, "no_invalid")
    bad = np.frombuffer(lab, np.uint16).copy()
    bad[[17, 2097151]] = value
    with pytest.raises(IndexError):
        sk.occupancy(bad.tobytes(), inv, lm)
    with pytest.raises(ValueError, match=r"b\.label: 2 voxel labels are at or past the remap table's 359 entries"):
        targets.semantic_kitti_occupancy([lab, bad.tobytes()], [inv, inv], lm,
                                         names=[("a.label", "a.invalid"), ("b.label", "b.invalid")])
    # the last in-table value is an unknown key: 255, no error
    ok = np.frombuffer(lab, np.uint16).copy()
    ok[17] = 358
    assert int(targets.semantic_kitti_occupancy(ok.tobytes(), inv, lm).view(-1)[17]) == 255


def test_staging_buffer_reused_across_batch_sizes(cuda, lm):
    """the pinned staging buffer grows and is reused: each call's volume is its own files', whatever came before"""
    frames = [sk.synthetic_voxels(lm, 80 + i, m) for i, m in enumerate(MODES)]
    ref = [sk.occupancy(lab, inv, lm) for lab, inv in frames]
    for sl in (slice(0, 1), slice(0, 4), slice(4, 5), slice(1, 5), slice(2, 3)):
        out = targets.semantic_kitti_occupancy([f[0] for f in frames[sl]], [f[1] for f in frames[sl]], lm).cpu().numpy()
        for b, r in enumerate(ref[sl]):
            assert np.array_equal(out[b], r), f"{MODES[sl][b]} after a reuse"


def test_one_launch_and_graph_replay(cuda, lm):
    frames = [sk.synthetic_voxels(lm, 30 + i, "mixed") for i in range(4)]
    lut = torch.from_numpy(targets.semkitti_remap_lut(lm)).to(cuda)
    label = torch.from_numpy(np.frombuffer(b"".join(f[0] for f in frames), np.uint8).copy()).to(cuda)
    invalid = torch.from_numpy(np.frombuffer(b"".join(f[1] for f in frames), np.uint8).copy()).to(cuda)
    counts = set()
    for B in (1, 4):
        n0 = ops.LAUNCH_COUNT[0]
        ops.semkitti_labels(label[:B * targets.SEMKITTI_LABEL_BYTES], invalid[:B * targets.SEMKITTI_INVALID_BYTES], B,
                            sk.NVOX, lut)
        counts.add(ops.LAUNCH_COUNT[0] - n0)
    assert counts == {1}
    outs = []
    graph_replay(lambda: outs.extend(ops.semkitti_labels(label, invalid, 4, sk.NVOX, lut)), outs)
    vol, bad = outs
    assert int(bad.abs().sum()) == 0
    for b, (lab, inv) in enumerate(frames):
        assert np.array_equal(vol[b].view(256, 256, 32).cpu().numpy(), sk.occupancy(lab, inv, lm))


def test_misaligned_labels_are_refused(cuda, lm):
    from util import misaligned, rejected
    lut = torch.from_numpy(targets.semkitti_remap_lut(lm)).to(cuda)
    label = torch.zeros(targets.SEMKITTI_LABEL_BYTES + 16, dtype=torch.uint8, device=cuda)
    invalid = torch.zeros(targets.SEMKITTI_INVALID_BYTES, dtype=torch.uint8, device=cuda)
    out = torch.zeros((1, sk.NVOX), dtype=torch.int64, device=cuda)
    bad = torch.zeros(1, dtype=torch.int32, device=cuda)
    rejected("occ_semkitti_labels", misaligned(label), invalid, 1, sk.NVOX, lut, lut.numel(), bad, out,
             buffers=(out, bad))
    rejected("occ_semkitti_labels", label, invalid, 1, sk.NVOX - 4, lut, lut.numel(), bad, out, buffers=(out, bad))


# ---------------------------------------------------------------------------------------------- the detector
def test_detector_targets_from_voxel_files(cuda, lm, tmp_path):
    from test_gpu_detector import detector, inputs
    from occformer_b200 import dist_eval
    model, _ = detector("kitti", cuda)
    frames = [sk.synthetic_voxels(lm, 50 + b, "mixed") for b in range(2)]
    host = torch.from_numpy(np.stack([sk.occupancy(lab, inv, lm) for lab, inv in frames])).to(cuda)

    def voxels(b):
        return dict(label=frames[b][0], invalid=frames[b][1], files=[f"{b}.label", f"{b}.invalid"], learning_map=lm)

    metas, img_inputs, _, _ = inputs("kitti", 2, cuda)
    assert torch.equal(model.occupancy_targets(None, [dict(m, semkitti_voxels=voxels(b)) for b, m in
                                                      enumerate(metas)]), host)

    metas, img_inputs, _, _ = inputs("kitti", 1, cuda)
    ref = model.simple_test(metas, img_inputs, gt_occ=host[:1])
    assert model.simple_test(metas, img_inputs)["target_voxels"] is None  # unchanged without the files
    with_files = [dict(metas[0], semkitti_voxels=voxels(0))]
    out = model.simple_test(with_files, img_inputs)
    assert torch.equal(out["target_voxels"], host[:1])
    given = host[:1]
    assert model.simple_test(with_files, img_inputs, gt_occ=given)["target_voxels"] is given
    assert set(out) == set(ref)
    # the SSC counts of this run's output against the device-built targets == against the gt_occ of the reference's
    # path: the preprocessing's float32 .npy, loaded as LoadSemKittiAnnotation does and collated to the device
    npy = os.path.join(str(tmp_path), "000000_1_1.npy")
    np.save(npy, sk.occupancy(*frames[0], lm).astype(np.float32))
    gt_occ = torch.tensor(np.load(npy)).long()[None].to(cuda)
    assert torch.equal(out["target_voxels"], gt_occ)
    a, b = (dist_eval.ssc_counts(out["output_labels"], t.to(torch.uint8), 20) for t in (out["target_voxels"], gt_occ))
    assert torch.equal(a, b)
    # and == the host's count (torch.bincount) of the same output against the npy-loaded volume
    host_counts = dist_eval.ssc_counts(out["output_labels"].cpu(), torch.tensor(np.load(npy)).long()[None], 20)
    assert torch.equal(a.cpu(), host_counts)
    assert int(a[3:].sum()) > 0
