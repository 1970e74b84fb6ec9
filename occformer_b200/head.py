"""H100-native Mask2Former-3D occupancy decoder heads, drop-in for the reference's

    HEADS 'Mask2FormerNuscOccHead'          projects/mmdet3d_plugin/occformer/mask2former/mask2former_nusc_occ.py:23-745
    HEADS 'Mask2FormerOccHead' (KITTI)      .../mask2former/mask2former_occ.py (same forward, :569-671; no lidarseg)
    HEADS 'Mask2FormerNuscPanopticOccHead'  .../mask2former/mask2former_nusc_panoptic_occ.py (same forward, :613-713)
    POSITIONAL_ENCODING 'SinePositionalEncoding3D'  .../positional_encodings/positional_encoding.py:11-108
    mmcv 1.4.0 DetrTransformerDecoder / BaseTransformerLayer / MultiheadAttention / FFN (parameter containers only)

Same constructor kwargs, same ``forward(voxel_feats, img_metas) -> (cls_pred_list, mask_pred_list)`` and
``simple_test(voxel_feats, img_metas, points=None) -> {'output_voxels': [...], 'output_points': ...}``, same
``state_dict`` keys (SURVEY.md Appendix B).  Inference only: losses / assigner / point sampling (training side,
RNG driven; SURVEY.md 8(a) A18-A19) are not part of this path and ``forward_train`` raises.

All arithmetic runs in libocc_b200.so: wgmma GEMMs on split-bf16 operands (three passes, fp32-faithful) for the
voxel-side contractions (K/V projections of the three memories, batched over the layers that share a level;
mask_embed x mask_feature einsum; masked cross attention) and fused fp32 kernels for the 100-query side
(csrc/head_ops.cu).  ``simple_test`` never materialises the reference's ten
(B,Q,X,Y,Z) mask tensors nor the upsampled (B,Q,*occ_size) logits: masks live query-last (B,S,Q), are pooled /
thresholded in place, and the final upsample + sigmoid + class mix (semantic heads) or upsample + argmax + id
numbering (panoptic head) runs in CUDA kernels.

Up to 256 queries.  The kernels run Qs = round_up(num_queries, 4) query slots per sample so that every query-last row
stays 16-byte aligned; the padded slots start from zero query_feat / query_embed rows, never act as self-attention
keys, get zero class probabilities and are cut from every returned tensor.
"""
import math

import torch
import torch.nn as nn

from . import ops
from .common import PreparedModule, twin_of
from .dist_eval import PanopticEval
from .registry import HEADS, POSITIONAL_ENCODING


def _get(cfg, key, default=None):
    if cfg is None:
        return default
    if isinstance(cfg, dict):
        return cfg.get(key, default)
    return getattr(cfg, key, default)


# ------------------------------------------------------------------------------------------ parameter containers
class _MHA(nn.Module):
    """torch.nn.MultiheadAttention parameter layout (packed in_proj)."""

    def __init__(self, E):
        super().__init__()
        self.in_proj_weight = nn.Parameter(torch.empty(3 * E, E))
        self.in_proj_bias = nn.Parameter(torch.zeros(3 * E))
        self.out_proj = nn.Linear(E, E)
        nn.init.xavier_uniform_(self.in_proj_weight)


class _Attn(nn.Module):  # mmcv MultiheadAttention wrapper: .attn
    def __init__(self, E):
        super().__init__()
        self.attn = _MHA(E)


class _FFN(nn.Module):  # mmcv FFN: layers = Sequential(Sequential(Linear, act, Dropout), Linear, Dropout)
    def __init__(self, E, F):
        super().__init__()
        self.layers = nn.Sequential(nn.Sequential(nn.Linear(E, F), nn.ReLU(inplace=True), nn.Dropout(0.0)),
                                    nn.Linear(F, E), nn.Dropout(0.0))


class _DecoderLayer(nn.Module):
    def __init__(self, E, F):
        super().__init__()
        self.attentions = nn.ModuleList([_Attn(E), _Attn(E)])  # 0 = cross, 1 = self
        self.ffns = nn.ModuleList([_FFN(E, F)])
        self.norms = nn.ModuleList([nn.LayerNorm(E) for _ in range(3)])


class _Decoder(nn.Module):
    def __init__(self, E, F, L):
        super().__init__()
        self.layers = nn.ModuleList([_DecoderLayer(E, F) for _ in range(L)])
        self.post_norm = nn.LayerNorm(E)
        self.embed_dims = E


@POSITIONAL_ENCODING.register_module()
class SinePositionalEncoding3D(nn.Module):
    """positional_encoding.py:11-108 with an all-False mask: the encoding depends on the grid size only, so it is
    computed once per size by occ_sine_pos3d and cached."""

    def __init__(self, num_feats, temperature=10000, normalize=False, scale=2 * math.pi, eps=1e-6, offset=0.0, **kw):
        super().__init__()
        assert normalize, "the reference configs use normalize=True"
        self.num_feats, self.temperature, self.scale, self.eps, self.offset = int(num_feats), temperature, scale, eps, offset
        self._cache = {}

    def rows(self, X, Y, Z, device):
        key = (X, Y, Z, str(device))
        if key not in self._cache:
            self._cache[key] = ops.sine_pos3d(X, Y, Z, self.num_feats, device, float(self.temperature), float(self.scale),
                                              float(self.eps), float(self.offset))
        return self._cache[key]

    def forward(self, mask):
        B, X, Y, Z = mask.shape
        r = self.rows(X, Y, Z, mask.device)
        return r.view(1, X, Y, Z, -1).permute(0, 4, 1, 2, 3).expand(B, -1, -1, -1, -1)


# ------------------------------------------------------------------------------------------ the head
class _Mask2FormerOccBase(PreparedModule):
    lidarseg = False

    def __init__(self, feat_channels, out_channels, num_occupancy_classes=20, num_queries=100,
                 num_transformer_feat_level=3, enforce_decoder_input_project=False, transformer_decoder=None,
                 positional_encoding=None, pooling_attn_mask=True, point_cloud_range=None, padding_mode="border",
                 sample_weight_gamma=0.25,
                 loss_cls=None, loss_mask=None, loss_dice=None, train_cfg=None, test_cfg=None, init_cfg=None, **kwargs):
        super().__init__()
        self.num_occupancy_classes = self.num_classes = num_occupancy_classes
        self.num_queries = num_queries
        self.point_cloud_range = point_cloud_range
        self.num_transformer_feat_level = num_transformer_feat_level
        tl = _get(transformer_decoder, "transformerlayers")
        attn_cfgs = _get(tl, "attn_cfgs")
        if isinstance(attn_cfgs, (list, tuple)):
            attn_cfgs = attn_cfgs[0]
        self.num_heads = int(_get(attn_cfgs, "num_heads"))
        E = int(_get(attn_cfgs, "embed_dims", feat_channels))
        self.num_transformer_decoder_layers = int(_get(transformer_decoder, "num_layers"))
        order = tuple(_get(tl, "operation_order", ("cross_attn", "norm", "self_attn", "norm", "ffn", "norm")))
        if order != ("cross_attn", "norm", "self_attn", "norm", "ffn", "norm"):
            raise NotImplementedError(f"occformer_b200: operation_order {order} (the reference configs use the post-norm "
                                      "cross/self/ffn order)")
        F = _get(tl, "feedforward_channels") or _get(_get(tl, "ffn_cfgs"), "feedforward_channels", 8 * E)
        self.ffn_channels = int(F)
        self.decoder_embed_dims = E
        if E != feat_channels or enforce_decoder_input_project or out_channels != feat_channels:
            raise NotImplementedError("occformer_b200: decoder_input_projs other than Identity (feat_channels == embed_dims "
                                      "in every reference config, mask2former_nusc_occ.py:99-106)")
        if E != self.num_heads * 32 or E % 32 or E > 256 or not 0 < num_queries <= 256:
            raise NotImplementedError("occformer_b200: head kernels are built for head_dim 32, embed_dims <= 256, "
                                      "num_queries <= 256")
        self.num_slots = (num_queries + 3) // 4 * 4
        if not pooling_attn_mask:
            raise NotImplementedError("occformer_b200: pooling_attn_mask=False (trilinear attn-mask downsampling)")
        self.transformer_decoder = _Decoder(E, self.ffn_channels, self.num_transformer_decoder_layers)
        self.decoder_input_projs = nn.ModuleList([nn.Identity() for _ in range(num_transformer_feat_level)])
        pe = dict(positional_encoding or dict(num_feats=E // 3, normalize=True))
        pe.pop("type", None)
        self.decoder_positional_encoding = SinePositionalEncoding3D(**pe)
        assert 3 * self.decoder_positional_encoding.num_feats == E
        self.query_embed = nn.Embedding(num_queries, feat_channels)
        self.query_feat = nn.Embedding(num_queries, feat_channels)
        self.level_embed = nn.Embedding(num_transformer_feat_level, feat_channels)
        self.cls_embed = nn.Linear(feat_channels, self.num_classes + 1)
        self.mask_embed = nn.Sequential(nn.Linear(feat_channels, feat_channels), nn.ReLU(inplace=True),
                                        nn.Linear(feat_channels, feat_channels), nn.ReLU(inplace=True),
                                        nn.Linear(feat_channels, out_channels))
        self.test_cfg, self.train_cfg = test_cfg, train_cfg
        self.pooling_attn_mask = pooling_attn_mask
        self.sample_weight_gamma = sample_weight_gamma
        self.align_corners = True
        self.padding_mode = padding_mode

    # ------------------------------------------------------------------ one-time weight preparation
    @torch.no_grad()
    def _prepare(self):
        E, nl, L = self.decoder_embed_dims, self.num_transformer_feat_level, self.num_transformer_decoder_layers
        T = lambda w: w.detach().float().t().contiguous()  # noqa: E731  (out,in) -> K-major (in,out)
        V = lambda w: w.detach().float().contiguous()      # noqa: E731
        dec = self.transformer_decoder
        P = {"head": dict(pn_w=V(dec.post_norm.weight), pn_b=V(dec.post_norm.bias), clsT=T(self.cls_embed.weight),
                          cls_b=V(self.cls_embed.bias), m0T=T(self.mask_embed[0].weight), m0b=V(self.mask_embed[0].bias),
                          m1T=T(self.mask_embed[2].weight), m1b=V(self.mask_embed[2].bias),
                          m2T=T(self.mask_embed[4].weight), m2b=V(self.mask_embed[4].bias)),
             "layers": [], "level_embed": V(self.level_embed.weight), "query_pos": self._slots(self.query_embed.weight),
             "query_feat": self._slots(self.query_feat.weight)}
        slots = {}
        kw = [[] for _ in range(nl)]
        kb = [[] for _ in range(nl)]
        vw = [[] for _ in range(nl)]
        vb = [[] for _ in range(nl)]
        for i, layer in enumerate(dec.layers):
            ca, sa = layer.attentions[0].attn, layer.attentions[1].attn
            lvl = i % nl
            slots[i] = len(kw[lvl])
            kw[lvl].append(ca.in_proj_weight[E:2 * E]); kb[lvl].append(ca.in_proj_bias[E:2 * E])
            vw[lvl].append(ca.in_proj_weight[2 * E:]); vb[lvl].append(ca.in_proj_bias[2 * E:])
            ffn = layer.ffns[0].layers
            P["layers"].append(dict(
                ca_wqT=T(ca.in_proj_weight[:E]), ca_bq=V(ca.in_proj_bias[:E]), ca_woT=T(ca.out_proj.weight),
                ca_bo=V(ca.out_proj.bias), n0w=V(layer.norms[0].weight), n0b=V(layer.norms[0].bias),
                sa_inT=T(sa.in_proj_weight), sa_inb=V(sa.in_proj_bias), sa_woT=T(sa.out_proj.weight),
                sa_bo=V(sa.out_proj.bias), n1w=V(layer.norms[1].weight), n1b=V(layer.norms[1].bias),
                f1T=T(ffn[0][0].weight), f1b=V(ffn[0][0].bias), f2T=T(ffn[1].weight), f2b=V(ffn[1].bias),
                n2w=V(layer.norms[2].weight), n2b=V(layer.norms[2].bias)))
        P["slots"] = slots
        cat = lambda ts: torch.cat([t.detach().float() for t in ts], 0).contiguous()  # noqa: E731
        P["kw"] = [ops.split_weight(cat(w)) if w else None for w in kw]
        P["vw"] = [ops.split_weight(cat(w)) if w else None for w in vw]
        P["kb"] = [cat(b) if b else None for b in kb]
        P["vb"] = [cat(b) if b else None for b in vb]
        return P

    def _slots(self, w):
        """(Q, E) query parameter -> (Qs, E) fp32 rows, the padded slots zero"""
        out = w.detach().float().new_zeros((self.num_slots, w.shape[1]))
        out[:w.shape[0]] = w.detach().float()
        return out

    # ------------------------------------------------------------------ layout helpers
    @staticmethod
    def _query_last(mask_preds):
        """reference-layout (B,Q,X,Y,Z) logits -> query-last (B,S,Qs) fp32, slots >= Q zero"""
        B, Q = mask_preds.shape[:2]
        m = mask_preds.float().reshape(B, Q, -1).permute(0, 2, 1)
        Qs = (Q + 3) // 4 * 4
        if Qs == Q:
            return m.contiguous()
        out = m.new_zeros((B, m.shape[1], Qs))
        out[..., :Q] = m
        return out

    @staticmethod
    def _rows(t):
        """(B,C,X,Y,Z) tensor of any strides -> (kernel input, channel_last flag).  Zero-copy both for contiguous
        reference-layout tensors and for permuted views of channel-last memory (what this package hands around)."""
        if not t.is_cuda:
            raise RuntimeError("occformer_b200: the decoder head runs on CUDA tensors only (no CPU fallback)")
        t = t.float()
        B, C, X, Y, Z = t.shape
        cl = t.permute(0, 2, 3, 4, 1)
        if cl.is_contiguous():
            return cl.reshape(B, X * Y * Z, C), True
        return t.contiguous().view(B, C, X * Y * Z), False

    # ------------------------------------------------------------------ the decoder
    @torch.no_grad()
    def _decode(self, voxel_feats, keep_all_masks):
        P = self.prepared()
        # Q = query slots of the kernels (rows per sample); Qr = real queries
        E, Q, Qr, H = self.decoder_embed_dims, self.num_slots, self.num_queries, self.num_heads
        nl, L, NC = self.num_transformer_feat_level, self.num_transformer_decoder_layers, self.num_classes + 1
        mf = voxel_feats[0]
        mems = voxel_feats[:0:-1]
        B = mf.shape[0]
        grid = tuple(mf.shape[-3:])
        V = grid[0] * grid[1] * grid[2]
        scale = 32 ** -0.5
        # mask features: channel-last S32, produced once (operand of the 1+L mask GEMMs); the neck of this package hands
        # the S32 twin over directly
        twin = twin_of(mf)
        if twin is not None:
            mf_r = twin.view(B, V, E)
        else:
            x, cl = self._rows(mf)
            mf_r, _ = ops.head_prep(x, cl)
        # memories: + level embed (+ positional encoding for K); K/V of every layer sharing the level in one GEMM each
        sizes, Kp, Vp, lds = [], [], [], []
        for l in range(nl):
            x, cl = self._rows(mems[l])
            g = tuple(mems[l].shape[-3:])
            sizes.append(g)
            pos = self.decoder_positional_encoding.rows(*g, x.device)
            mem_r, kpos_r = ops.head_prep(x, cl, P["level_embed"][l], pos)
            S = g[0] * g[1] * g[2]
            if P["kw"][l] is None:
                Kp.append(None), Vp.append(None), lds.append(0)
                continue
            # S32 outputs (one chunk per (key, head)): tensor-core operands of the cross-attention kernel
            Kp.append(ops.gemm(kpos_r.view(B * S, E), P["kw"][l], bias=P["kb"][l], split_out=True))
            Vp.append(ops.gemm(mem_r.view(B * S, E), P["vw"][l], bias=P["vb"][l], split_out=True))
            lds.append(P["kw"][l].shape[0])
        query = P["query_feat"].unsqueeze(0).expand(B, Q, E).reshape(B * Q, E).contiguous()
        qpos = P["query_pos"]

        def forward_head(query_in, target, keep_mask, norm2=None, next_layer=None, ffn_part=None):
            nq = None
            if next_layer is not None:
                Ln = P["layers"][next_layer]
                nq = (qpos, Q, Ln["ca_wqT"], Ln["ca_bq"], scale)
            cls, membed, query, qh = ops.query_head(query_in, P["head"], NC, norm2=norm2, next_q=nq, ffn_part=ffn_part)
            mask, pf = None, None
            if target is not None and not keep_mask:
                # einsum + adaptive max pool + threshold bookkeeping in one kernel, the (B,V,Q) logits never written
                pf = ops.mask_gemm_pool(mf_r, membed, B, grid, target, Q)
            if pf is not None:
                pooled, flag = pf
            else:
                mask = torch.empty((B, V, Q), dtype=torch.float32, device=query_in.device)
                for b in range(B):
                    ops.gemm(mf_r[b], membed[b * Q:(b + 1) * Q], out=mask[b])
                pooled, flag = ops.mask_pool(mask, B, grid, target, Q) if target is not None else (None, None)
            return cls.view(B, Q, NC)[:, :Qr], mask, pooled, flag, query, qh

        cls_list, mask_list = [], []
        cls, mask, pooled, flag, query, qh = forward_head(query, sizes[0], keep_all_masks or L == 0,
                                                          next_layer=0 if L > 0 else None)
        cls_list.append(cls)
        if keep_all_masks or L == 0:
            mask_list.append(mask)
        for i in range(L):
            lvl = i % nl
            S = sizes[lvl][0] * sizes[lvl][1] * sizes[lvl][2]
            Lw = P["layers"][i]
            off = P["slots"][i] * E
            part, nchunk = ops.cross_attn_tc(qh, Kp[lvl], Vp[lvl], lds[lvl], off, off, pooled, flag, B, S, Q, E, H)
            q1, sa = ops.cross_merge(part, nchunk, H, query, qpos, Q, Lw, scale)
            ybuf, ffn_part = ops.self_attn_ffn(sa, q1, Q, Lw, H, nkeys=Qr)
            last = i == L - 1
            cls, mask, pooled, flag, query, qh = forward_head(ybuf, None if last else sizes[(i + 1) % nl],
                                                              keep_all_masks or last, norm2=(Lw["n2w"], Lw["n2b"]),
                                                              next_layer=None if last else i + 1, ffn_part=ffn_part)
            cls_list.append(cls)
            if keep_all_masks or last:
                mask_list.append(mask)
        return cls_list, mask_list, grid

    def forward(self, voxel_feats, img_metas=None, **kwargs):
        """-> (cls_pred_list[1+L] of (B,Q,K+1), mask_pred_list[1+L] of (B,Q,X,Y,Z))  (mask2former_nusc_occ.py:589-689)"""
        cls_list, masks, grid = self._decode(voxel_feats, keep_all_masks=True)
        B, Q, Qs = cls_list[0].shape[0], self.num_queries, self.num_slots
        V = grid[0] * grid[1] * grid[2]
        masks = [ops.transpose_sq(m, B, V, Qs).view(B, Qs, *grid) for m in masks]
        if Qs != Q:
            masks = [m[:, :Q].contiguous() for m in masks]
        return cls_list, masks

    def format_results(self, mask_cls_results, mask_pred_results):
        """mask2former_nusc_occ.py:691-696 on reference-layout tensors (B,Q,K+1), (B,Q,X,Y,Z)."""
        B, Q, NC = mask_cls_results.shape
        grid = tuple(mask_pred_results.shape[-3:])
        return ops.classmix(self._query_last(mask_pred_results), mask_cls_results.float().contiguous(), B, grid, grid, Q, NC)

    @torch.no_grad()
    def simple_test(self, voxel_feats, img_metas, points=None, **kwargs):
        """mask2former_nusc_occ.py:698-745 -> {'output_voxels': [(B,K,*occ_size)], 'output_points': (sum n, K) | None}"""
        cls_list, masks, grid = self._decode(voxel_feats, keep_all_masks=False)
        cls, mask = cls_list[-1].contiguous(), masks[-1]
        B, Q, NC = cls.shape
        occ_size = tuple(int(v) for v in img_metas[0]["occ_size"])
        out, labels = ops.classmix(mask, cls, B, grid, occ_size, Q, NC, with_labels=True)
        # 'output_labels' is an addition to the reference's dict: argmax over classes (what its evaluation loop
        # derives from output_voxels, occupancyformer.py:238-243), produced by the same kernel
        res = {"output_voxels": [out], "output_points": None, "output_labels": labels}
        if self.lidarseg and points is not None:
            res["output_points"] = self.forward_lidarseg(cls, mask, points, img_metas, _grid=grid,
                                                         _native=out if occ_size == grid else None)
        return res

    @torch.no_grad()
    def forward_lidarseg(self, cls_preds, mask_preds, points, img_metas=None, _grid=None, _native=None):
        """mask2former_nusc_occ.py:505-542, eval branch.  mask_preds: (B,Q,X,Y,Z) reference layout, or the internal
        query-last (B,S,Q) tensor together with _grid."""
        B, Q, NC = cls_preds.shape
        if _grid is None:
            _grid = tuple(mask_preds.shape[-3:])
            mask_preds = self._query_last(mask_preds)
        vox = _native if _native is not None else ops.classmix(mask_preds, cls_preds.float().contiguous(), B, _grid, _grid, Q, NC)
        pc_range = img_metas[0]["pc_range"] if img_metas is not None else self.point_cloud_range
        outs = [ops.lidarseg_points(vox[b], pts.to(vox.device), pc_range, border=self.padding_mode == "border")
                for b, pts in enumerate(points)]
        return torch.cat(outs, dim=0)

    def get_sampling_weights(self):
        """mask2former_occ.py:158-166: class-frequency sampling weights ** gamma (KITTI heads; the nuScenes head samples
        LiDAR points instead)."""
        from . import sampling
        self.sample_weights = sampling.class_sampling_weights(sampling.SEMANTIC_KITTI_CLASS_FREQUENCIES,
                                                              self.sample_weight_gamma)
        return self.sample_weights

    def forward_train(self, *a, **k):
        raise NotImplementedError(
            "occformer_b200 covers the inference forward (SURVEY.md section 8).  The training step (losses, Hungarian "
            "assigner) stays in the reference plugin; its class-guided point sampling (SURVEY.md A18 / A19) is available as "
            "host functions under the reference names in occformer_b200.sampling, and forward() / simple_test() of this head "
            "return the same cls / mask predictions the reference's loss code consumes.")


@HEADS.register_module()
class Mask2FormerNuscOccHead(_Mask2FormerOccBase):
    lidarseg = True


@HEADS.register_module()
class Mask2FormerOccHead(_Mask2FormerOccBase):
    lidarseg = False


@HEADS.register_module()
class Mask2FormerNuscPanopticOccHead(_Mask2FormerOccBase):
    """Same decoder forward (mask2former_nusc_panoptic_occ.py:613-713); panoptic inference (:715-835) on the GPU.

    ``simple_test`` returns the reference's dict: ``output_voxels = [(semantic, panoptic)]`` (int64 (B, *occ_size)),
    ``output_points`` / ``output_panoptic_points`` (int64 (B, N), None without points; every sample needs the same point
    count, as the reference stacks them).  A voxel / point takes the class of its highest-logit query; a thing class's
    panoptic id is label * 1000 + the instance number of its (label, query) pair, a stuff class's label * 1000.  The
    per-query numbering runs on the device (occ_panoptic_voxels / occ_panoptic_points): no host synchronisation, so the
    whole call can be captured in a CUDA graph."""
    lidarseg = True

    def __init__(self, *args, stuff_indices=None, thing_indices=None, **kwargs):
        super().__init__(*args, **kwargs)
        self.stuff_indices = stuff_indices
        self.thing_indices = thing_indices
        self._thing = ops.thing_mask(thing_indices)
        self.panoptic_metric = PanopticEval(self.num_classes, ignore=[0], min_points=15)  # reference :148

    @torch.no_grad()
    def simple_test(self, voxel_feats, img_metas, points=None, **kwargs):
        """mask2former_nusc_panoptic_occ.py:786-835"""
        cls_list, masks, grid = self._decode(voxel_feats, keep_all_masks=False)
        cls, mask = cls_list[-1].contiguous(), masks[-1]
        B, Q = cls.shape[:2]
        occ_size = tuple(int(v) for v in img_metas[0]["occ_size"])
        res = {"output_voxels": [ops.panoptic_voxels(mask, cls, B, grid, occ_size, Q, self._thing)],
               "output_points": None, "output_panoptic_points": None}
        if points is not None:
            res["output_points"], res["output_panoptic_points"] = self.forward_lidar_panopticseg(
                cls, mask, points, img_metas, _grid=grid)
        return res

    @torch.no_grad()
    def format_panoptic_occupancy_results(self, mask_cls_results, mask_pred_results):
        """:749-784 on reference-layout (B,Q,K+1), (B,Q,X,Y,Z) -> (semantic, panoptic) int64 (B,X,Y,Z)"""
        B, Q, _ = mask_cls_results.shape
        grid = tuple(mask_pred_results.shape[-3:])
        return ops.panoptic_voxels(self._query_last(mask_pred_results), mask_cls_results.float().contiguous(), B, grid,
                                   grid, Q, self._thing)

    @torch.no_grad()
    def format_panoptic_lidar_results(self, mask_cls_results, mask_pred_results):
        """:715-747 on (B,Q,K+1) class logits and (B,Q,N) point logits -> (semantic, panoptic) int64 (B,N)"""
        B, Q, _ = mask_cls_results.shape
        n = mask_pred_results.shape[-1]
        sem, pan = ops.panoptic_voxels(self._query_last(mask_pred_results.reshape(B, Q, n, 1, 1)),
                                       mask_cls_results.float().contiguous(), B, (n, 1, 1), (n, 1, 1), Q, self._thing,
                                       point_rule=True)
        return sem.view(B, n), pan.view(B, n)

    @torch.no_grad()
    def forward_lidar_panopticseg(self, cls_preds, mask_preds, points, img_metas=None, _grid=None):
        """:515-563, eval branch: (semantic, panoptic) int64 (B, N) of the LiDAR points.  mask_preds: (B,Q,X,Y,Z)
        reference layout, or the internal query-last (B,S,Qs) tensor together with _grid."""
        B, Q, _ = cls_preds.shape
        if _grid is None:
            _grid = tuple(mask_preds.shape[-3:])
            mask_preds = self._query_last(mask_preds)
        pc_range = img_metas[0]["pc_range"] if img_metas is not None else self.point_cloud_range
        pts = torch.stack([p.to(mask_preds.device)[:, :3].float() for p in points])
        return ops.panoptic_points(mask_preds, cls_preds.float().contiguous(), B, _grid, Q, self._thing, pts, pc_range,
                                   border=self.padding_mode == "border")


def head_cfg(E, Q, K, num_layers, num_heads, pc_range, num_levels=3, ffn=None):
    """The head section of the reference configs (occformer_nusc_r50_256x704.py:132-190), inference-relevant keys."""
    return dict(feat_channels=E, out_channels=E, num_queries=Q, num_occupancy_classes=K,
                num_transformer_feat_level=num_levels, pooling_attn_mask=True,
                positional_encoding=dict(type="SinePositionalEncoding3D", num_feats=E / 3, normalize=True),
                transformer_decoder=dict(type="DetrTransformerDecoder", return_intermediate=True, num_layers=num_layers,
                                         transformerlayers=dict(
                                             type="DetrTransformerDecoderLayer",
                                             attn_cfgs=dict(type="MultiheadAttention", embed_dims=E, num_heads=num_heads),
                                             feedforward_channels=ffn or 8 * E,
                                             operation_order=("cross_attn", "norm", "self_attn", "norm", "ffn", "norm"))),
                point_cloud_range=pc_range)


def build_nusc_head(E, Q, K, num_layers, num_heads, pc_range, num_levels=3, ffn=None):
    return Mask2FormerNuscOccHead(**head_cfg(E, Q, K, num_layers, num_heads, pc_range, num_levels, ffn))
