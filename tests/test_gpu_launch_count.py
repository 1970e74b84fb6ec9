"""The library's launch counter (occ_launch_count, ops.LAUNCH_COUNT, bench.py's gpu_launches) against the GPU's own
record: one connected step on the PR1 grid (1 camera 128x128 -> 50x50x8 voxels -> the reference-width encoder, neck and
head simple_test) under torch.profiler.  Every kernel of the library lives in namespace occ, so the count must equal the
occ:: kernels plus the memsets of the trace (torch issues none in this step)."""
import pytest
import torch

from util import trace
from occformer_b200 import synth

pytestmark = pytest.mark.gpu


class _PassThroughDepthNet(torch.nn.Module):
    def forward(self, x, mlp_input=None):
        return x


def _pr1_step(cuda):
    """-> a function running one connected forward step on the PR1 grid through the registered modules"""
    from occformer_b200 import BACKBONES, HEADS, NECKS
    from occformer_b200.head import head_cfg
    from occformer_b200.neck import neck_cfg
    planes, nums, strides = [128, 256, 512, 1024], [2, 2, 2, 2], [1, 2, 2, 2]
    E, Q, K, L = 192, 100, 17, 9
    pc = [-20.0, -20.0, -2.0, 20.0, 20.0, 4.4]
    vt = NECKS.build(dict(type="ViewTransformerLiftSplatShootVoxel", grid_config=synth.grid_config("pr1"),
                          data_config={"input_size": (128, 128)}, numC_input=112 + 128, numC_Trans=128,
                          depth_net=_PassThroughDepthNet())).to(cuda)
    enc = BACKBONES.build(dict(type="OccupancyEncoder", in_channels=128, num_stage=4, block_numbers=nums,
                               block_inplanes=planes, block_strides=strides, out_indices=(0, 1, 2, 3),
                               norm_cfg=dict(type="GN", num_groups=32, requires_grad=True), with_cp=True))
    enc.load_state_dict(synth.make_encoder_state(128, planes, nums, strides, seed=0), strict=True)
    neck = NECKS.build(dict(type="MSDeformAttnPixelDecoder3D", **neck_cfg(planes, [2, 4, 8, 16], E, 6, 8, 3, 4, 4 * E)))
    neck.load_state_dict(synth.make_neck_state(planes, E, 6, 8, 3, 4, 4 * E, seed=2), strict=True)
    head = HEADS.build(dict(type="Mask2FormerNuscOccHead", **head_cfg(E, Q, K, L, E // 32, pc)))
    head.load_state_dict(synth.make_head_state(E, Q, K, L, 3, seed=1), strict=True)
    enc, neck, head = enc.to(cuda).eval(), neck.to(cuda).eval(), head.to(cuda).eval()
    dd, feat = synth.lift_inputs(1, 1, 112, 8, 8, 128, seed=0)
    x = torch.cat([dd, feat], dim=1).view(1, 1, 112 + 128, 8, 8).to(cuda)
    cams = synth.pr1_camera(1)
    inp = [x] + [cams[k].to(cuda) for k in ("rots", "trans", "intrins", "post_rots", "post_trans", "bda")] + [None]
    metas = [dict(occ_size=[100, 100, 16], pc_range=pc)]

    @torch.no_grad()
    def step():
        voxel, _ = vt(inp)
        return head.simple_test(neck(enc(voxel)), metas)

    return step


def test_launch_count_matches_profiler_trace(cuda):
    step = _pr1_step(cuda)
    step()  # warm-up: lazy weight packing, workspaces, module loading
    t = trace(step)
    print(f"[launch count] counted {t['counted']}, trace: {t['kernels']} occ:: kernels + {t['memsets']} memsets")
    assert t["kernels"] > 0 and t["memsets"] > 0
    assert t["counted"] == t["kernels"] + t["memsets"]
