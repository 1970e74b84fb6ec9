"""H100-native 3-D multi-scale deformable-attention pixel decoder, drop-in for the reference's

    NECKS 'MSDeformAttnPixelDecoder3D'              projects/mmdet3d_plugin/occformer/necks/multiscale_deformattn_3d.py:20-249
    ATTENTION 'MultiScaleDeformableAttention3D'     projects/mmdet3d_plugin/occformer/necks/multi_scale_deform_attn_3d.py:83-286
    mmcv 1.4.0 ConvModule / BaseTransformerLayer / FFN / DetrTransformerEncoder (parameter containers only)

Same constructor kwargs (cfg section ``img_bev_encoder_neck`` of occformer_nusc_r50_256x704.py:98-131), same
``forward(feats: list of (B,C_i,X_i,Y_i,Z_i), high -> low resolution) -> [mask_feature, memory level 2, 1, 0]`` and the same
``state_dict`` keys.  SURVEY.md 8(f)1: the caller between the two starred subsystems -- with it the forward is connected
(encoder pyramid -> neck -> head).

All arithmetic runs in libocc_b200.so: the 1x1x1 / 3x3x3 convolutions and the value / offset projections of every
encoder layer on the wgmma GEMM (split-bf16 operands, three passes, fp32-faithful), the deformable gather / token
preparation / FPN up-sampling in csrc/neck_ops.cu, and the rest of every encoder layer (output projection, both
LayerNorms, FFN; E = 96 or 192) as one kernel in csrc/neck_tail_fused.cu.  Tokens are kept level-major (csrc/neck_ops.cu) so that no concatenation, split or transpose of the
reference's forward exists here; tensors that feed a contraction travel in the S32 split format and carry over from the
encoder / to the head as S32 twins (common.attach_twin).  Inference only.
"""
import torch
import torch.nn as nn

from . import ops
from .common import PreparedModule, attach_twin, twin_of
from .head import SinePositionalEncoding3D, _get
from .registry import ATTENTION, NECKS


class _ConvGN(nn.Module):
    """mmcv ConvModule(conv -> GN [-> act]) parameter container: .conv, .gn"""

    def __init__(self, cin, cout, k, bias, groups):
        super().__init__()
        self.conv = nn.Conv3d(cin, cout, k, padding=k // 2, bias=bias)
        self.gn = nn.GroupNorm(groups, cout)


@ATTENTION.register_module()
class MultiScaleDeformableAttention3D(nn.Module):
    """Parameter container with the reference's names (multi_scale_deform_attn_3d.py:128-183); the arithmetic lives in
    MSDeformAttnPixelDecoder3D.forward (fused projections + occ_ms_deform_attn)."""

    def __init__(self, embed_dims=256, num_heads=8, num_levels=4, num_points=4, im2col_step=64, dropout=0.1, batch_first=False,
                 norm_cfg=None, init_cfg=None, **kw):
        super().__init__()
        if embed_dims % num_heads:
            raise ValueError("embed_dims must be divisible by num_heads")
        self.embed_dims, self.num_heads, self.num_levels, self.num_points = embed_dims, num_heads, num_levels, num_points
        self.sampling_offsets = nn.Linear(embed_dims, num_heads * num_levels * num_points * 3)
        self.attention_weights = nn.Linear(embed_dims, num_heads * num_levels * num_points)
        self.value_proj = nn.Linear(embed_dims, embed_dims)
        self.output_proj = nn.Linear(embed_dims, embed_dims)


class _FFN(nn.Module):
    def __init__(self, E, F):
        super().__init__()
        self.layers = nn.Sequential(nn.Sequential(nn.Linear(E, F), nn.ReLU(inplace=True), nn.Dropout(0.0)),
                                    nn.Linear(F, E), nn.Dropout(0.0))


class _EncoderLayer(nn.Module):
    def __init__(self, attn_cfg, E, F):
        super().__init__()
        self.attentions = nn.ModuleList([MultiScaleDeformableAttention3D(**attn_cfg)])
        self.ffns = nn.ModuleList([_FFN(E, F)])
        self.norms = nn.ModuleList([nn.LayerNorm(E), nn.LayerNorm(E)])


class _Encoder(nn.Module):
    def __init__(self, attn_cfg, E, F, L):
        super().__init__()
        self.layers = nn.ModuleList([_EncoderLayer(attn_cfg, E, F) for _ in range(L)])


@NECKS.register_module()
class MSDeformAttnPixelDecoder3D(PreparedModule):
    def __init__(self, in_channels=[256, 512, 1024, 2048], strides=[4, 8, 16, 32], feat_channels=256, out_channels=256,
                 num_outs=3, conv_cfg=None, norm_cfg=None, act_cfg=None, encoder=None, positional_encoding=None,
                 init_cfg=None, **kwargs):
        super().__init__()
        norm_cfg = dict(norm_cfg or dict(type="GN", num_groups=32))
        if norm_cfg.get("type", "GN") != "GN":
            raise NotImplementedError("occformer_b200: the neck implements the reference's GN configuration")
        G = norm_cfg.get("num_groups", 32)
        tl = _get(encoder, "transformerlayers")
        attn = _get(tl, "attn_cfgs")
        if isinstance(attn, (list, tuple)):
            attn = attn[0]
        order = tuple(_get(tl, "operation_order", ("self_attn", "norm", "ffn", "norm")))
        if order != ("self_attn", "norm", "ffn", "norm"):
            raise NotImplementedError(f"occformer_b200: operation_order {order}")
        E = feat_channels
        attn_cfg = dict(embed_dims=int(_get(attn, "embed_dims", E)), num_heads=int(_get(attn, "num_heads", 8)),
                        num_levels=int(_get(attn, "num_levels", 3)), num_points=int(_get(attn, "num_points", 4)))
        if attn_cfg["embed_dims"] != E or E % 32 or (E // attn_cfg["num_heads"]) % 4:
            raise NotImplementedError("occformer_b200: neck kernels need embed_dims == feat_channels, a multiple of 32, and a "
                                      "head dim that is a multiple of 4")
        F = int(_get(tl, "feedforward_channels") or _get(_get(tl, "ffn_cfgs"), "feedforward_channels", 4 * E))
        self.strides = list(strides)
        self.in_channels = list(in_channels)
        self.num_input_levels = len(in_channels)
        self.num_encoder_levels = attn_cfg["num_levels"]
        self.num_heads, self.num_points, self.embed_dims, self.groups = attn_cfg["num_heads"], attn_cfg["num_points"], E, G
        nin, L = self.num_input_levels, self.num_encoder_levels
        self.input_convs = nn.ModuleList([_ConvGN(in_channels[i], E, 1, True, G) for i in range(nin - 1, nin - L - 1, -1)])
        self.encoder = _Encoder(attn_cfg, E, F, int(_get(encoder, "num_layers", 6)))
        pe = dict(positional_encoding or dict(num_feats=E // 3, normalize=True))
        pe.pop("type", None)
        self.postional_encoding = SinePositionalEncoding3D(**pe)  # (sic) the reference's attribute name
        self.level_encoding = nn.Embedding(L, E)
        self.lateral_convs = nn.ModuleList([_ConvGN(in_channels[i], E, 1, False, G) for i in range(nin - L - 1, -1, -1)])
        self.output_convs = nn.ModuleList([_ConvGN(E, E, 3, False, G) for i in range(nin - L - 1, -1, -1)])
        self.mask_feature = nn.Conv3d(E, out_channels, 1)
        self.num_outs = num_outs

    @torch.no_grad()
    def _prepare(self):
        sw = ops.split_weight
        P = {"in": [], "layers": [], "lat": [], "out": [], "pos": {}}
        for m in self.input_convs:
            P["in"].append(ops.repack_conv_weight(m.conv.weight)[0])
        for lyr in self.encoder.layers:
            a = lyr.attentions[0]
            ffn = lyr.ffns[0].layers
            # value_proj rows padded per head to a 128-byte slice (24 -> 32 floats at the reference width): the gather
            # kernel is bound by the number of distinct lines it touches
            wv_p, bv_p = ops.pad_head_rows(a.value_proj.weight, a.value_proj.bias, a.num_heads)
            P["layers"].append(dict(
                wv=sw(wv_p), bv=bv_p, wo=sw(a.output_proj.weight),
                # sampling offsets and attention logits of a token come from ONE GEMM: N = H*L*P*3 + H*L*P
                wow=sw(torch.cat([a.sampling_offsets.weight.detach().float(), a.attention_weights.weight.detach().float()], 0)),
                bow=torch.cat([a.sampling_offsets.bias.detach().float(), a.attention_weights.bias.detach().float()], 0).contiguous(),
                w1=sw(ffn[0][0].weight), w2=sw(ffn[1].weight)))
        for m in self.lateral_convs:
            P["lat"].append(ops.repack_conv_weight(m.conv.weight)[0])
        for m in self.output_convs:
            P["out"].append(ops.repack_conv_weight(m.conv.weight))
        P["mf"] = ops.repack_conv_weight(self.mask_feature.weight)[0]
        return P

    def _pos_rows(self, P, grids, device):
        """query_pos of the encoder (:160-163): sine encoding of every level + its level embedding, (Nq, E), cached per
        grid in P["pos"]"""
        key = (tuple(grids), str(device))
        if key not in P["pos"]:
            rows = [self.postional_encoding.rows(*g, device) + self.level_encoding.weight[i].detach().float()
                    for i, g in enumerate(grids)]
            P["pos"][key] = torch.cat(rows, 0).contiguous()
        return P["pos"][key]

    @staticmethod
    def _operand(f):
        """(B,C,X,Y,Z) reference-layout tensor -> its channel-last S32 twin (picked up from the encoder, else split here)"""
        if not f.is_cuda:
            raise RuntimeError("occformer_b200: the neck runs on CUDA tensors only (no CPU fallback)")
        twin = twin_of(f)
        if twin is not None:
            return twin
        return ops.to_split(f.float().permute(0, 2, 3, 4, 1).contiguous())

    @torch.no_grad()
    def forward(self, feats):
        P = self.prepared()
        nin, L, E, G, H = self.num_input_levels, self.num_encoder_levels, self.embed_dims, self.groups, self.num_heads
        B = feats[0].shape[0]
        dev = feats[0].device
        grids = [tuple(feats[nin - i - 1].shape[-3:]) for i in range(L)]  # coarse -> fine
        ns = [g[0] * g[1] * g[2] for g in grids]
        starts = [sum(ns[:i]) for i in range(L)]
        Nq = sum(ns)
        # ---- input convs (1x1x1 + bias, GN, no activation) straight into the level-major token tensor (:152-157)
        x = torch.empty((B * Nq, E), dtype=torch.float32, device=dev)
        for i in range(L):
            m = self.input_convs[i]
            raw = ops.conv(self._operand(feats[nin - i - 1]), P["in"][i], (1, 1, 1), bias=m.conv.bias)
            st = ops.gn_stats(raw.view(B * ns[i], E), B, ns[i], E, G)
            ops.gn_apply(raw.view(B * ns[i], E), st, m.gn.weight, m.gn.bias, ns[i], G, relu=False,
                         out_f32=x[B * starts[i]:B * (starts[i] + ns[i])])
        pos = self._pos_rows(P, grids, dev)
        strides = [self.strides[nin - i - 1] for i in range(L)]
        _, x_s, xq_s = ops.neck_token_prep(x, grids, B, pos=pos, want_f32=False, want_pos=True)
        # ---- DetrTransformerEncoder of BaseTransformerLayer('self_attn', 'norm', 'ffn', 'norm')  (:203-215)
        nl = len(self.encoder.layers)
        for li, (lyr, W) in enumerate(zip(self.encoder.layers, P["layers"])):
            a, ffn = lyr.attentions[0], lyr.ffns[0].layers
            v = ops.gemm(x_s, W["wv"], bias=W["bv"])
            ow = ops.gemm(xq_s, W["wow"], bias=W["bow"])
            att = ops.ms_deform_attn(v, ow, grids, strides, B, E, H, self.num_points)
            # output_proj + residual, norms[0], FFN + residual, norms[1]: one kernel, nothing in between crosses HBM
            last = li == nl - 1
            x, x_s, xq_s = ops.neck_layer_tail(att, x, W["wo"], a.output_proj.bias, (lyr.norms[0].weight, lyr.norms[0].bias),
                                               W["w1"], ffn[0][0].bias, W["w2"], ffn[1].bias,
                                               (lyr.norms[1].weight, lyr.norms[1].bias), grids, B, pos=pos,
                                               want_s32=not last, want_pos=not last)
        # ---- the encoder output of every level is a contiguous channel-last tensor (:217-226)
        outs = [x[B * starts[i]:B * (starts[i] + ns[i])].view(B, *grids[i], E) for i in range(L)]
        # ---- FPN path for the levels that skipped the encoder (:228-246)
        mf_s = None
        for i in range(nin - L - 1, -1, -1):
            lat, oc = self.lateral_convs[i], self.output_convs[i]
            # GroupNorm statistics of both convs ride in their epilogues
            st = torch.zeros(B, G, 2, dtype=torch.float64, device=dev)
            cur = ops.conv(self._operand(feats[i]), P["lat"][i], (1, 1, 1), gn_stats=st, cpg=E // G)
            Bc, X, Y, Z, _ = cur.shape
            y_s = ops.gn_upsample_add(cur, st, lat.gn.weight, lat.gn.bias, G, outs[-1])
            w3, k3 = P["out"][i]
            st = torch.zeros(B, G, 2, dtype=torch.float64, device=dev)
            o_raw = ops.conv(y_s, w3, k3, gn_stats=st, cpg=E // G)
            need_f32 = i > 0  # a finer FPN level up-samples it; the finest one only feeds mask_feature
            o, o_s = ops.gn_apply(o_raw.view(-1, E), st, oc.gn.weight, oc.gn.bias, X * Y * Z, G, relu=True,
                                  want_f32=need_f32, want_split=True)
            outs.append(o.view(B, X, Y, Z, E) if o is not None else None)
            mf_s = o_s.view(B, X, Y, Z, E)
        if mf_s is None:  # every level went through the encoder: mask_feature acts on the finest encoder level
            mf_s = ops.to_split(outs[-1])
        mf = ops.conv(mf_s, P["mf"], (1, 1, 1), bias=self.mask_feature.bias)
        outs[-1] = mf
        res = [o.permute(0, 4, 1, 2, 3) for o in outs[::-1]]
        attach_twin(res[0], ops.to_split(mf))  # operand of the head's 1 + L mask GEMMs
        return res


def neck_cfg(in_channels, strides, E, num_layers, num_heads, num_levels, num_points, ffn):
    """The ``img_bev_encoder_neck`` section of the reference configs (occformer_nusc_r50_256x704.py:98-131)."""
    return dict(in_channels=list(in_channels), strides=list(strides), feat_channels=E, out_channels=E, num_outs=3,
                norm_cfg=dict(type="GN", num_groups=32), act_cfg=dict(type="ReLU"),
                encoder=dict(type="DetrTransformerEncoder", num_layers=num_layers,
                             transformerlayers=dict(
                                 type="BaseTransformerLayer",
                                 attn_cfgs=dict(type="MultiScaleDeformableAttention3D", embed_dims=E, num_heads=num_heads,
                                                num_levels=num_levels, num_points=num_points, im2col_step=64, dropout=0.0,
                                                batch_first=False, norm_cfg=None, init_cfg=None),
                                 ffn_cfgs=dict(embed_dims=E), feedforward_channels=ffn, ffn_dropout=0.0,
                                 operation_order=("self_attn", "norm", "ffn", "norm")),
                             init_cfg=None),
                positional_encoding=dict(type="SinePositionalEncoding3D", num_feats=E // 3, normalize=True))
