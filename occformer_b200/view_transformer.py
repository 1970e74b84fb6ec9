"""H100-native LSS lift-splat view transformer, drop-in for

    NECKS 'ViewTransformerLiftSplatShootVoxel'   projects/mmdet3d_plugin/occformer/image2bev/ViewTransformerLSSVoxel.py:12-121
    (geometry / frustum parts of its bases)      .../image2bev/ViewTransformerLSSBEVDepth.py:21-25,64-150
    mmdet3d.ops.bev_pool.bev_pool                mmdetection3d/mmdet3d/ops/bev_pool/bev_pool.py:83-97

``forward`` never materialises the (B,N,D,fH,fW,C) volume: depth softmax and NCHW->NHWC happen in a small
prologue and the pooling kernel multiplies depth and context on the fly.  ``voxel_pooling(geom, volume)`` and
``bev_pool(feats, coords, ...)`` keep the reference's materialised-input signatures for callers that use them.

The constructor follows the reference chain ViewTransformerLiftSplatShoot -> ViewTransformerLSSBEVDepth ->
ViewTransformerLiftSplatShootVoxel (ViewTransformerLSSBEVDepth.py:64-99,565-576; ViewTransformerLSSVoxel.py:12-25): same
kwargs, ``depth_net = DepthNet(numC_input, numC_input, numC_Trans, D, cam_channels)`` with the reference's state_dict
keys (occformer_b200/depthnet.py: this package's kernels on CUDA tensors, SURVEY.md 8(f)3), ``get_mlp_input``, ``get_depth_loss``.
``depth_net=`` (an extension) substitutes another module, e.g. a pass-through when the caller already holds
post-DepthNet maps.  ``forward`` is inference-only (no autograd through the pooling kernels).
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import ops
from .common import PreparedModule, attach_twin
from .depthnet import DepthNet
from .registry import NECKS


def gen_dx_bx(xbound, ybound, zbound):
    """ViewTransformerLSSBEVDepth.py:21-25 (float32 torch.Tensor arithmetic, kept as is for bit-exactness)."""
    dx = torch.Tensor([row[2] for row in [xbound, ybound, zbound]])
    bx = torch.Tensor([row[0] + row[2] / 2.0 for row in [xbound, ybound, zbound]])
    nx = torch.Tensor([(row[1] - row[0]) / row[2] for row in [xbound, ybound, zbound]])
    return dx, bx, nx


def bev_pool(feats, coords, B, D, H, W):
    """Drop-in for mmdet3d.ops.bev_pool.bev_pool: feats (n,C) fp32 CUDA, coords (n,4) integer (x,y,z,b);
    B, D(=nz), H(=nx), W(=ny) ints or 0-d tensors.  Returns (B, C, D, H, W) (a permuted view of the
    channel-last grid; values identical to the reference's contiguous tensor).  Forward only."""
    assert feats.shape[0] == coords.shape[0]
    B, D, H, W = int(B), int(D), int(H), int(W)
    out = ops.bev_pool_channel_last(feats.float().contiguous(), coords.long().contiguous(), B, H, W, D)
    return out.permute(0, 4, 3, 1, 2)  # (B,X,Y,Z,C) -> (B,C,Z,X,Y)


@NECKS.register_module()
class ViewTransformerLiftSplatShootVoxel(PreparedModule):
    def __init__(self, loss_depth_weight=1.0, grid_config=None, data_config=None, numC_input=512, numC_Trans=64,
                 downsample=16, point_cloud_range=None, loss_depth_type="bce", cam_channels=27, loss_depth_reg_weight=0.0,
                 use_voxel_net=False, accelerate=False, use_bev_pool=True, vp_megvii=False, vp_stero=False,
                 depth_net=None, **kwargs):
        super().__init__()
        if grid_config is None:
            grid_config = {"xbound": [-51.2, 51.2, 0.8], "ybound": [-51.2, 51.2, 0.8], "zbound": [-10.0, 10.0, 20.0],
                           "dbound": [1.0, 60.0, 1.0]}
        if use_voxel_net or accelerate or vp_megvii or vp_stero:
            raise NotImplementedError("occformer_b200: use_voxel_net / accelerate / vp_megvii / vp_stero are off in every "
                                      "OccFormer config (occformer_nusc_r50_256x704.py:79-85) and are not built")
        self.grid_config = grid_config
        dx, bx, nx = gen_dx_bx(grid_config["xbound"], grid_config["ybound"], grid_config["zbound"])
        self.dx = nn.Parameter(dx, requires_grad=False)
        self.bx = nn.Parameter(bx, requires_grad=False)
        self.nx = nn.Parameter(nx, requires_grad=False)
        self.data_config = data_config or {"input_size": (256, 704)}
        self.downsample = downsample
        self.frustum = self.create_frustum()
        self.D = self.frustum.shape[0]
        self.numC_input, self.numC_Trans = numC_input, numC_Trans
        self.cam_channels = cam_channels
        # ViewTransformerLSSBEVDepth.py:571-572; ``depth_net=`` replaces it (the signature is decided here, once)
        self.depth_net = depth_net if depth_net is not None else DepthNet(numC_input, numC_input, numC_Trans, self.D,
                                                                          cam_channels=cam_channels)
        self._depth_net_takes_mlp = not isinstance(self.depth_net, nn.Conv2d)
        self.depth_aggregation_net = None
        self.loss_depth_weight = loss_depth_weight
        self.loss_depth_reg_weight = loss_depth_reg_weight
        self.loss_depth_type = loss_depth_type
        self.cam_depth_range = grid_config["dbound"]
        self.point_cloud_range = point_cloud_range
        self.geom_feats = None
        self.accelerate, self.use_bev_pool, self.vp_megvii, self.vp_stereo = accelerate, use_bev_pool, vp_megvii, vp_stero

    def _prepare(self):
        """(dx, bx, nx) as host float lists, the by-value arguments of the pooling kernels (one D2H)"""
        return (self.dx.detach().cpu().tolist(), self.bx.detach().cpu().tolist(), self.nx.detach().cpu().tolist())

    _host_params = PreparedModule.prepared  # the name bench.py reads them by

    def grid_size(self):
        _, _, nx = self.prepared()
        return int(nx[0]), int(nx[1]), int(nx[2])

    def create_frustum(self):
        """ViewTransformerLSSBEVDepth.py:104-115"""
        ogfH, ogfW = self.data_config["input_size"]
        fH, fW = ogfH // self.downsample, ogfW // self.downsample
        ds = torch.arange(*self.grid_config["dbound"], dtype=torch.float).view(-1, 1, 1).expand(-1, fH, fW)
        D = ds.shape[0]
        xs = torch.linspace(0, ogfW - 1, fW, dtype=torch.float).view(1, 1, fW).expand(D, fH, fW)
        ys = torch.linspace(0, ogfH - 1, fH, dtype=torch.float).view(1, fH, 1).expand(D, fH, fW)
        return nn.Parameter(torch.stack((xs, ys, ds), -1), requires_grad=False)

    def get_geometry(self, rots, trans, intrins, post_rots, post_trans, bda):
        """ViewTransformerLSSBEVDepth.py:117-150 as one fused kernel (occ_lss_geometry): (B,N,D,fH,fW,3) ego points."""
        if not trans.is_cuda:
            raise RuntimeError("occformer_b200: get_geometry runs on CUDA tensors only (no CPU fallback)")
        return ops.lss_geometry(self.frustum.data, rots, trans, intrins, post_rots, post_trans, bda)

    def get_mlp_input(self, rot, tran, intrin, post_rot, post_tran, bda=None):
        """ViewTransformerLSSBEVDepth.py:591-646 -- the camera-aware MLP input (B, N, 27) (33 for KITTI's 3x4 / 4x4
        intrinsics with a 4x4 bda): selected entries of intrinsics / post-transform / bda followed by the flattened
        sensor-to-ego [R|t].  Host-side tensor indexing (a few hundred bytes), same dtype/device as the inputs."""
        B, N = rot.shape[:2]
        if bda is None:
            bda = torch.eye(3).to(rot).view(1, 3, 3).repeat(B, 1, 1)
        bda = bda.view(B, 1, *bda.shape[-2:]).repeat(1, N, 1, 1)
        cols = [intrin[:, :, 0, 0], intrin[:, :, 1, 1], intrin[:, :, 0, 2], intrin[:, :, 1, 2]]
        if intrin.shape[-1] == 4:
            cols += [intrin[:, :, 0, 3], intrin[:, :, 1, 3], intrin[:, :, 2, 3]]
        cols += [post_rot[:, :, 0, 0], post_rot[:, :, 0, 1], post_tran[:, :, 0], post_rot[:, :, 1, 0], post_rot[:, :, 1, 1],
                 post_tran[:, :, 1], bda[:, :, 0, 0], bda[:, :, 0, 1], bda[:, :, 1, 0], bda[:, :, 1, 1], bda[:, :, 2, 2]]
        mlp_input = torch.stack(cols, dim=-1)
        if intrin.shape[-1] == 4 and bda.shape[-1] == 4:
            mlp_input = torch.cat((mlp_input, bda[:, :, :3, -1]), dim=2)
        sensor2ego = torch.cat([rot, tran.reshape(B, N, 3, 1)], dim=-1).reshape(B, N, -1)
        return torch.cat([mlp_input, sensor2ego], dim=-1)

    def get_depth_dist(self, x):
        return x.softmax(dim=1)

    # ------------------------------------------------------------------ training-side helpers (host torch, as the reference)
    def get_downsampled_gt_depth(self, gt_depths):
        """ViewTransformerLSSVoxel.py:27-51: (B,N,H,W) LiDAR depth maps -> (depth bin values (B*N,h,w), one-hot (B*N*h*w, D))."""
        B, N, H, W = gt_depths.shape
        ds = self.downsample
        g = gt_depths.view(B * N, H // ds, ds, W // ds, ds, 1).permute(0, 1, 3, 5, 2, 4).contiguous().view(-1, ds * ds)
        g = torch.where(g == 0.0, 1e5 * torch.ones_like(g), g).min(dim=-1).values.view(B * N, H // ds, W // ds)
        db = self.grid_config["dbound"]
        g = (g - (db[0] - db[2] / 2)) / db[2]
        vals = g.clone()
        g = torch.where((g < self.D + 1) & (g >= 0.0), g, torch.zeros_like(g))
        onehot = F.one_hot(g.long(), num_classes=self.D + 1).view(-1, self.D + 1)[:, 1:]
        return vals, onehot.float()

    def get_bce_depth_loss(self, depth_labels, depth_preds):
        """ViewTransformerLSSVoxel.py:53-66"""
        _, depth_labels = self.get_downsampled_gt_depth(depth_labels)
        depth_preds = depth_preds.permute(0, 2, 3, 1).contiguous().view(-1, self.D)
        fg = depth_labels.max(dim=1).values > 0.0
        loss = F.binary_cross_entropy(depth_preds[fg].float(), depth_labels[fg], reduction="none").sum()
        return loss / max(1.0, float(fg.sum()))

    def get_depth_loss(self, depth_labels, depth_preds):
        """ViewTransformerLSSVoxel.py:68-75"""
        if self.loss_depth_type != "bce":
            raise NotImplementedError(f"loss_depth_type {self.loss_depth_type!r} (the reference implements 'bce' only)")
        return self.loss_depth_weight * self.get_bce_depth_loss(depth_labels, depth_preds)

    # ------------------------------------------------------------------ the hot path
    @torch.no_grad()
    def voxel_pooling(self, geom_feats, x):
        """ViewTransformerLSSVoxel.py:77-100 with a materialised volume x (B,N,D,H,W,C).  -> (B,C,X,Y,Z) view."""
        B, N, D, H, W, C = x.shape
        dx, bx, nx = self.prepared()
        feats = x.reshape(B * N * D * H * W, C).float().contiguous()
        geom = geom_feats.reshape(-1, 3).float().contiguous()
        out = ops.voxel_pool_geom(feats, geom, B, dx, bx, nx, self.grid_size())
        return out.permute(0, 4, 1, 2, 3)

    @torch.no_grad()
    def lift_splat(self, depth_digit, img_feat, geom, B, N, with_split=False):
        """Fused lift-splat on post-DepthNet tensors: depth logits (B*N,D,fH,fW), context (B*N,C,fH,fW),
        geom (B,N,D,fH,fW,3).  Returns (channel-last grid (B,X,Y,Z,C) [or (grid, S32 twin) when with_split], depth_prob)."""
        dx, bx, nx = self.prepared()
        prob, feat_cl = ops.lift_prologue(depth_digit.float().contiguous(), img_feat.float().contiguous())
        grid = ops.lift_splat(prob, feat_cl, geom.float().contiguous(), B, N, dx, bx, nx, self.grid_size(),
                              with_split=with_split)
        return grid, prob

    @torch.no_grad()
    def forward(self, input):
        """ViewTransformerLSSVoxel.py:102-121: returns (bev_feat (B,C,X,Y,Z), depth_prob (B*N,D,fH,fW)).  Inference only:
        runs under no_grad (the pooling kernels have no backward)."""
        (x, rots, trans, intrins, post_rots, post_trans, bda, mlp_input) = input[:8]
        B, N, C, H, W = x.shape
        x = x.view(B * N, C, H, W)
        x = self.depth_net(x, mlp_input) if self._depth_net_takes_mlp else self.depth_net(x)
        depth_digit = x[:, :self.D, ...]
        img_feat = x[:, self.D:self.D + self.numC_Trans, ...]
        if not x.is_cuda:
            raise RuntimeError("occformer_b200: the view transformer runs on CUDA tensors only (no CPU fallback)")
        # depth softmax + get_geometry + voxel index + point lists + NHWC transpose in ONE front kernel, then the pooling
        # kernel (occ_lift_splat_fused); get_geometry / lift_splat stay available as separate calls
        split = self.numC_Trans % 32 == 0
        dx, bx, nx = self.prepared()
        grid, depth_prob = ops.lift_splat_fused(depth_digit, img_feat, self.frustum.data, rots, trans, intrins, post_rots, post_trans, bda, B, N,
                                                dx, bx, nx, self.grid_size(), with_split=split)
        if split:
            # the S32 twin is the operand of the encoder's first conv (occformer_b200.encoder picks it up)
            return attach_twin(grid[0].permute(0, 4, 1, 2, 3), grid[1]), depth_prob
        return grid.permute(0, 4, 1, 2, 3), depth_prob
