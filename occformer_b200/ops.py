"""Torch-tensor wrappers over the C-ABI kernels (device memory + streams are torch's; the math is ours).

Every call checks each tensor argument against its pointer declaration in include/occ_b200.h (CUDA, current device,
dtype, contiguity), passes raw pointers and the current torch stream to libocc_b200.so and raises RuntimeError on a
non-zero return code.  No fallback paths.
"""
import ctypes

import numpy as np
import torch

from ._lib import check, lib, parameters


class _LaunchCount:
    """``LAUNCH_COUNT[0]``: kernel launches and memsets the library has enqueued in this process (occ_launch_count;
    bench.py reports it as gpu_launches)."""

    def __getitem__(self, i):
        if i != 0:
            raise IndexError(i)
        return lib().occ_launch_count()


LAUNCH_COUNT = _LaunchCount()


def _stream():
    """the current torch stream of the current device (where _checked requires a call's tensors to live)"""
    return torch.cuda.current_stream().cuda_stream


# ----------------------------------------------------------------------------------------------- host-side caches
_stream_ws = {}      # (kernel, device, stream) -> (grow-only uint8 workspace, superseded workspaces)
_device_tables = {}  # (device, key) -> constant table on the device


def _stream_workspace(kernel, dev, nbytes):
    """kernel's grow-only uint8 workspace for the current stream of dev, at least nbytes long"""
    key = (kernel, str(dev), torch.cuda.current_stream(dev).cuda_stream)
    ent = _stream_ws.get(key)
    if ent is None or ent[0].numel() < nbytes:
        # a graph captured before the workspace grew still points at the old one: keep it referenced
        old = [] if ent is None else ent[1] + [ent[0]]
        ent = (torch.empty(nbytes, dtype=torch.uint8, device=dev), old)
        _stream_ws[key] = ent
    return ent[0]


def _device_table(dev, key, make):
    """the device copy of the numpy array make() returns, built on first use per (dev, key); key stands for the content"""
    k = (str(dev), key)
    t = _device_tables.get(k)
    if t is None:
        t = torch.from_numpy(make()).to(dev)
        _device_tables[k] = t
    return t


def _stage(pieces):
    """bytes-like pieces -> (uint8 CUDA buffer of the current device holding them back to back, each piece's byte
    offset): one pinned host buffer, which torch's caching host allocator recycles once the copy is done, and one
    host-to-device copy"""
    offsets = np.cumsum([0] + [len(f) for f in pieces]).tolist()
    host = torch.empty(offsets[-1], dtype=torch.uint8, pin_memory=True)
    hv = host.numpy()
    for f, o in zip(pieces, offsets):
        hv[o:o + len(f)] = np.frombuffer(f, np.uint8)
    return host.to(torch.cuda.current_device(), non_blocking=True), offsets[:-1]


# tensor dtype per pointee type of the header (S32 is a float32 container; void: any; size_t* is host-only: no tensor)
_DTYPES = {"float": torch.float32, "double": torch.float64, "long long": torch.int64, "int": torch.int32,
           "unsigned": torch.int32, "unsigned int": torch.int32, "unsigned char": torch.uint8, "void": None}


def _checked(t, fn, i, strided=False):
    """tensor t as parameter i of fn, checked against its declaration in the header: a pointer whose pointee type matches
    t's dtype, t a contiguous (unless strided: the caller passes its strides) CUDA tensor on the current device -> t"""
    param, pointee = parameters()[fn][i]
    what = f"occformer_b200: {fn}({param})"
    if pointee not in _DTYPES:
        raise RuntimeError(f"{what} is not a device pointer and cannot take a tensor")
    if not t.is_cuda:
        raise RuntimeError(f"{what} must be a CUDA tensor (no CPU fallback exists)")
    if t.device.index != torch.cuda.current_device():
        raise RuntimeError(f"{what} lives on {t.device} but the current device is cuda:{torch.cuda.current_device()} "
                           "(wrap the call in torch.cuda.device(...))")
    if _DTYPES[pointee] not in (None, t.dtype):
        raise RuntimeError(f"{what} must be {_DTYPES[pointee]}, got {t.dtype}")
    if not (strided or t.is_contiguous()):
        raise RuntimeError(f"{what} must be contiguous")
    return t


def _call(name, *args, unsupported_ok=False):
    """lib().<name>(*args, current stream) with tensors checked and passed as device pointers and None as NULL -> its return
    code; raises RuntimeError if that is not 0 (or -2, unsupported shape with nothing enqueued, when unsupported_ok)"""
    args = [_checked(a, name, i).data_ptr() if torch.is_tensor(a) else a for i, a in enumerate(args)]
    rc = getattr(lib(), name)(*args, _stream())
    if not (unsupported_ok and rc == -2):
        check(rc, name)
    return rc


# ----------------------------------------------------------------------------------------------- S32 split format
# Operands of every tensor-core contraction are fp32 values stored as bf16 hi | lo halves per 32-column chunk (csrc/
# occ_ptx.cuh, include/occ_b200.h): same bytes and row pitch as the fp32 tensor, ~1e-5 relative error after the three
# bf16 passes.  Weights are split once at load time (torch ops below), activations by the producing kernel's epilogue.
def set_precision(mode):
    """"fp32" (default): every contraction in three bf16 tensor-core passes on hi/lo split operands (fp32-faithful, the
    mode of every parity claim).  "bf16": single pass on the hi halves (BASELINE config 5; ~3e-3 relative error per
    contraction, no reference twin).  Library-wide, takes effect for kernels launched afterwards.  Returns the old mode."""
    passes = {"fp32": 3, "bf16": 1}[mode]
    prev = lib().occ_set_mma_passes(passes)
    if prev < 0:
        raise RuntimeError("occ_set_mma_passes failed")
    return {3: "fp32", 1: "bf16"}[prev]


class precision:
    """``with ops.precision("bf16"): ...`` -- scoped set_precision."""

    def __init__(self, mode):
        self.mode = mode

    def __enter__(self):
        self.prev = set_precision(self.mode)
        return self

    def __exit__(self, *exc):
        set_precision(self.prev)
        return False


def split_weight(w):
    """(N, K) fp32 torch tensor (any device), K % 32 == 0 -> the same tensor in S32 (fp32 container, same shape)."""
    w = w.detach().float().contiguous()
    N, K = w.shape
    assert K % 32 == 0, f"S32 rows need K % 32 == 0, got {K}"
    hi = w.to(torch.bfloat16)
    lo = (w - hi.float()).to(torch.bfloat16)
    packed = torch.cat([hi.view(N, K // 32, 32), lo.view(N, K // 32, 32)], dim=2).contiguous()  # (N, K/32, 64) bf16
    return packed.view(torch.float32).reshape(N, K)


def unsplit_weight(ws):
    """inverse of split_weight (tests / debugging): S32 -> fp32 values hi + lo."""
    N, K = ws.shape
    p = ws.contiguous().view(torch.bfloat16).view(N, K // 32, 64).float()
    return (p[:, :, :32] + p[:, :, 32:]).reshape(N, K)


def to_split(x):
    """fp32 CUDA tensor (..., C), C % 32 == 0 -> S32 (device kernel)."""
    C = x.shape[-1]
    out = torch.empty_like(x)
    _call("occ_split_rows", x, out, x.numel() // C, C)
    return out


def from_split(x):
    C = x.shape[-1]
    out = torch.empty_like(x)
    _call("occ_unsplit_rows", x, out, x.numel() // C, C)
    return out


# ----------------------------------------------------------------------------------------------- voxel pooling
class VoxelPoolWorkspace:
    """View of the pooling workspace for one call with n_points points (bookkeeping left behind by the kernels)."""

    def __init__(self, buf, n_points, B, X, Y, Z):
        offs = [ctypes.c_size_t() for _ in range(4)]
        lib().occ_voxel_pool_workspace_layout(n_points, B, X, Y, Z, *[ctypes.byref(o) for o in offs])
        self.buf, self.nbytes = buf, buf.numel()
        self.off_counts, self.off_head, self.off_next, self.off_vox_id = (o.value for o in offs)
        self.V = B * X * Y * Z
        self.P = n_points

    def _ints(self, off, n):
        return self.buf[off:off + 4 * n].view(torch.int32)

    @property
    def counts(self):
        """points per voxel (= the reference's interval lengths)"""
        return self._ints(self.off_counts, self.V)

    @property
    def head(self):
        """first point (1-based id, 0 = empty) of every voxel's list"""
        return self._ints(self.off_head, self.V)

    @property
    def next(self):
        """next point (1-based id, 0 = end) of every kept point"""
        return self._ints(self.off_next, self.P)

    @property
    def vox_id(self):
        return self._ints(self.off_vox_id, self.P)


# (B, X, Y, Z, device) -> (uint8 buffer, point capacity, superseded buffers): one grow-only buffer per grid.  A CUDA
# graph captured before the buffer grew still points at the buffer it was captured with, so the superseded ones stay
# referenced.  Point capacities double, so the point arrays of all the superseded buffers together are no larger than
# the newest one's.
_ws_cache = {}


def _workspace(n_points, B, X, Y, Z, device):
    key = (B, X, Y, Z, str(device))
    n_points = max(int(n_points), 1)
    ent = _ws_cache.get(key)
    if ent is None or ent[1] < n_points:
        cap = 1 << (n_points - 1).bit_length()  # next power of two: the drop-in bev_pool sees a different n every sample
        nbytes = lib().occ_voxel_pool_workspace_bytes(cap, B, X, Y, Z)
        old = [] if ent is None else ent[2] + [ent[0]]
        ent = (torch.zeros(nbytes, dtype=torch.uint8, device=device), cap, old)
        _ws_cache[key] = ent
    return VoxelPoolWorkspace(ent[0], n_points, B, X, Y, Z)


_conv_ws = {}  # (device, stream) -> zeroed buffer: split-K ordering counters of occ_conv_bf16x3


def _conv_workspace(device):
    key = (str(device), torch.cuda.current_stream(device).cuda_stream)
    ws = _conv_ws.get(key)
    if ws is None:
        ws = torch.zeros(lib().occ_conv_workspace_bytes(), dtype=torch.uint8, device=device)
        _conv_ws[key] = ws
    return ws


def lss_geometry(frustum, rots, trans, intrins, post_rots, post_trans, bda):
    """frustum (D,fH,fW,3) + camera matrices -> geom (B,N,D,fH,fW,3)."""
    B, N = trans.shape[:2]
    D, fH, fW, _ = frustum.shape
    f = lambda t: t.float().contiguous()  # noqa: E731
    geom = torch.empty((B, N, D, fH, fW, 3), dtype=torch.float32, device=frustum.device)
    fr, r, t, k, pr, pt, bd = f(frustum), f(rots), f(trans), f(intrins), f(post_rots), f(post_trans), f(bda)
    _call("occ_lss_geometry", fr, D * fH * fW, r, t, k, k.shape[-2], k.shape[-1], pr, pt, bd, bd.shape[-1], B, N, geom)
    return geom


def lift_prologue(depth_logits, img_feat):
    """depth_logits (BN,D,fH,fW), img_feat (BN,C,fH,fW) -> depth_prob (BN,D,fH,fW), feat_cl (BN,fH*fW,C)."""
    BN, D, fH, fW = depth_logits.shape
    C = img_feat.shape[1]
    prob = torch.empty_like(depth_logits)
    feat_cl = torch.empty((BN, fH * fW, C), dtype=torch.float32, device=img_feat.device)
    _call("occ_lift_prologue", depth_logits, img_feat, prob, feat_cl, BN, D, C, fH * fW)
    return prob, feat_cl


def lift_splat(depth_prob, feat_cl, geom, B, N, dx, bx, nx, grid, return_workspace=False, with_split=False):
    """Fused lift-splat.  Returns the channel-last grid (B,X,Y,Z,C) [, its S32 copy when with_split]."""
    BN, D, fH, fW = depth_prob.shape
    C = feat_cl.shape[-1]
    X, Y, Z = grid
    P = B * N * D * fH * fW
    assert geom.numel() == 3 * P
    ws = _workspace(P, B, X, Y, Z, geom.device)
    out = torch.empty((B, X, Y, Z, C), dtype=torch.float32, device=geom.device)
    out_s = torch.empty_like(out) if with_split else None
    f = [float(v) for v in (*dx, *bx, *nx)]
    _call("occ_lift_splat", depth_prob, feat_cl, geom, out, out_s, B, N, D, fH * fW, C, *f, X, Y, Z, ws.buf, ws.nbytes)
    res = (out, out_s) if with_split else out
    return (res, ws) if return_workspace else res


def lift_splat_fused(depth_logits, img_feat, frustum, rots, trans, intrins, post_rots, post_trans, bda, B, N, dx, bx, nx,
                     grid, with_split=False):
    """The view transformer after DepthNet in three launches (memset, front kernel, pooling): depth_logits (BN,D,fH,fW),
    img_feat (BN,C,fH,fW) -> (grid (B,X,Y,Z,C) [, S32 twin], depth_prob (BN,D,fH,fW))."""
    BN, D, fH, fW = depth_logits.shape
    C = img_feat.shape[1]
    X, Y, Z = grid
    HW = fH * fW

    def plane(t, i):  # (BN, ch, fH, fW) fp32 whose cameras may be strided (channel slice of a bigger tensor): no copy
        t = t.float()
        if t.stride()[1:] != (HW, fW, 1):
            t = t.contiguous()
        return t, _checked(t, "occ_lift_splat_fused", i, strided=True).data_ptr(), t.stride(0)

    depth_logits, lp, ls = plane(depth_logits, 0)  # keeps a copy alive: the allocations below must not reuse it
    img_feat, fp, fs = plane(img_feat, 2)
    f = lambda t: t.float().contiguous()  # noqa: E731
    fr, r, t, k, pr, pt, bd = f(frustum), f(rots), f(trans), f(intrins), f(post_rots), f(post_trans), f(bda)
    dev = depth_logits.device
    ws = _workspace(BN * D * HW, B, X, Y, Z, dev)
    prob = torch.empty((BN, D, fH, fW), dtype=torch.float32, device=dev)
    feat_cl = torch.empty((BN, HW, C), dtype=torch.float32, device=dev)
    out = torch.empty((B, X, Y, Z, C), dtype=torch.float32, device=dev)
    out_s = torch.empty_like(out) if with_split else None
    fl = [float(v) for v in (*dx, *bx, *nx)]
    _call("occ_lift_splat_fused", lp, ls, fp, fs, fr, r, t, k, k.shape[-2], k.shape[-1], pr, pt, bd,
          bd.shape[-1], prob, feat_cl, out, out_s, B, N, D, HW, C, *fl, X, Y, Z, ws.buf, ws.nbytes)
    return ((out, out_s) if with_split else out), prob


def voxel_pool_geom(feats, geom, B, dx, bx, nx, grid, return_workspace=False):
    """Materialised-volume voxel pooling: feats (P,C), geom (P,3) -> (B,X,Y,Z,C)."""
    P_, C = feats.shape
    X, Y, Z = grid
    ws = _workspace(P_, B, X, Y, Z, feats.device)
    out = torch.empty((B, X, Y, Z, C), dtype=torch.float32, device=feats.device)
    f = [float(v) for v in (*dx, *bx, *nx)]
    _call("occ_voxel_pool_geom", feats, geom, out, B, P_ // B, C, *f, X, Y, Z, ws.buf, ws.nbytes)
    return (out, ws) if return_workspace else out


def bev_pool_channel_last(feats, coords, B, X, Y, Z, return_workspace=False):
    n, C = feats.shape
    ws = _workspace(n, B, X, Y, Z, feats.device)
    out = torch.empty((B, X, Y, Z, C), dtype=torch.float32, device=feats.device)
    _call("occ_bev_pool", feats, coords, out, n, C, B, X, Y, Z, ws.buf, ws.nbytes)
    return (out, ws) if return_workspace else out


# ----------------------------------------------------------------------------------------------- GEMM / conv
def gemm(a, w, bias=None, residual=None, act=0, split_out=False, out=None):
    """out[M,N] = act(a[M,K] @ w[N,K]^T + bias + residual), act 0 none, 1 ReLU, 2 GELU, 3 Swish: the residual is added
    before the activation.  a, w in S32
    (to_split / split_weight / a producer's split output); out fp32, or S32 when split_out (operand of the next
    contraction)."""
    M, K = a.shape
    N = w.shape[0]
    assert w.shape[1] == K
    if out is None:
        out = torch.empty((M, N), dtype=torch.float32, device=a.device)
    if residual is not None:
        assert residual.shape == (M, N)
    _call("occ_gemm_bf16x3", a, w, out, M, N, K, bias, residual, act, int(split_out))
    return out


def repack_conv_weight(w):
    """(Cout, Cin, kx, ky[, kz]) -> (Cout, taps*Cin) tap-major [(kx*KY + ky)*KZ + kz][cin] in S32 (Cin % 32 == 0)."""
    if w.dim() == 4:
        w = w.unsqueeze(-1)
    Cout, Cin, KX, KY, KZ = w.shape
    w2 = w.detach().float().permute(0, 2, 3, 4, 1).reshape(Cout, KX * KY * KZ * Cin)
    return split_weight(w2), (KX, KY, KZ)


def conv(x_cl, w2, ksize, stride=1, dil=1, bias=None, residual=None, act=0, split_out=False, gn_stats=None, cpg=0):
    """x_cl (B,X,Y,Z,Cin) channel-last S32; w2 from repack_conv_weight; returns (B,Xo,Yo,Zo,Cout) channel-last raw
    output (fp32, or S32 when split_out).  gn_stats: zero-initialised double tensor (B, groups, 2) receiving (sum, sumsq)
    of the raw output, cpg = Cout // groups channels per group (any cpg, at most 96 groups)."""
    B, X, Y, Z, Cin = x_cl.shape
    KX, KY, KZ = ksize
    Cout = w2.shape[0]
    assert w2.shape[1] == KX * KY * KZ * Cin

    def osz(n, k):
        p = dil * (k - 1) // 2
        return (n + 2 * p - dil * (k - 1) - 1) // stride + 1

    Xo, Yo, Zo = osz(X, KX), osz(Y, KY), osz(Z, KZ)
    out = torch.empty((B, Xo, Yo, Zo, Cout), dtype=torch.float32, device=x_cl.device)
    ws = _conv_workspace(x_cl.device)
    _call("occ_conv_bf16x3", x_cl, w2, out, B, X, Y, Z, Cin, Cout, KX, KY, KZ, stride, dil, bias, residual, act,
          int(split_out), gn_stats, cpg, ws, ws.numel())
    return out


def conv_into(x_cl, w2, ksize, out, out_off=0, dil=1, bias=None, residual=None, act=0, split_out=False):
    """Stride-1 "same" conv() written into columns [out_off, out_off + Cout) of out (B*X*Y*Z, ldo); the other columns
    are left as they are.  S32 output (split_out): ldo and out_off multiples of 32; fp32 output: multiples of 4.
    residual (B*X*Y*Z, Cout) contiguous.  -> out"""
    B, X, Y, Z, Cin = x_cl.shape
    KX, KY, KZ = ksize
    Cout = w2.shape[0]
    assert w2.shape[1] == KX * KY * KZ * Cin and out.dim() == 2 and out.shape[0] == B * X * Y * Z
    ws = _conv_workspace(x_cl.device)
    _call("occ_conv_slice_bf16x3", x_cl, w2, out, out.shape[1], out_off, B, X, Y, Z, Cin, Cout, KX, KY, KZ, 1, dil, bias,
          residual, act, int(split_out), None, 0, ws, ws.numel())
    return out


def conv_plan(B, X, Y, Z, Cin, Cout, ksize=(3, 3, 3), stride=1, dil=1, splitk_ok=True):
    """The tiling conv() picks for this shape: (tile rows, tile columns, ring stages, K splits).  splitk_ok=False for a
    conv with bias / residual / activation / split output (never split)."""
    plan = (ctypes.c_int * 4)()
    check(lib().occ_conv_plan(B, X, Y, Z, Cin, Cout, *ksize, stride, dil, int(splitk_ok), plan), "occ_conv_plan")
    return tuple(plan)


def conv_taps(x_cl, w2, taps, gn_stats=None, cpg=0):
    """Stride-1 convolution over an explicit tap table (several dilated branches in one launch): x_cl (B,X,Y,Z,Cin) S32,
    taps = [(dx, dy, dz), ...], w2 (Cout, len(taps)*Cin) S32 tap-major -> raw (B,X,Y,Z,Cout) fp32."""
    B, X, Y, Z, Cin = x_cl.shape
    Cout = w2.shape[0]
    assert w2.shape[1] == len(taps) * Cin
    out = torch.empty((B, X, Y, Z, Cout), dtype=torch.float32, device=x_cl.device)
    flat = [int(v) for t in taps for v in t]
    arr = (ctypes.c_int * len(flat))(*flat)
    _call("occ_conv_taps_bf16x3", x_cl, w2, out, B, X, Y, Z, Cin, Cout, len(taps), arr, gn_stats, cpg)
    return out


# ----------------------------------------------------------------------------------------------- DepthNet
def depthnet_cam_gates(mlp_in, w1T, b1, w2T, b2, wrT, br, weT, be):
    """mlp_in (n, cam) -> SE gates (2, n, C) of the depth (0) and context (1) chains; weights K-major, both chains
    stacked (occ_depthnet_cam_gates)."""
    n, cam = mlp_in.shape
    C = b1.shape[-1]
    gates = torch.empty((2, n, C), dtype=torch.float32, device=mlp_in.device)
    _call("occ_depthnet_cam_gates", mlp_in, cam, w1T, b1, w2T, b2, wrT, br, weT, be, gates, n, C)
    return gates


def se_apply(x, gates, n, rows_per_img):
    """x (n*rows_per_img, C) fp32, gates (2, n, C) -> (x*g_depth fp32, x*g_depth S32, x*g_ctx S32)."""
    C = x.shape[1]
    xd, xd_s, xc_s = torch.empty_like(x), torch.empty_like(x), torch.empty_like(x)
    _call("occ_se_apply", x, gates, xd, xd_s, xc_s, n, rows_per_img, C)
    return xd, xd_s, xc_s


def depthnet_gap_branch(x, w, b, cat, n, rows_per_img, out_off):
    """ASPP image-pooling branch of DepthNet: mean of x (n*rows_per_img, C) per image -> w (C, C) + b -> ReLU, broadcast
    into cat[:, out_off:out_off + C] (S32).  -> cat"""
    C = x.shape[1]
    ws = torch.empty((2, n, C), dtype=torch.float32, device=x.device)
    _call("occ_depthnet_gap_branch", x, ws, w, b, cat, n, rows_per_img, C, cat.shape[1], out_off)
    return cat


def deform_im2col(x_s, off, n, H, W, groups):
    """DCNv1 sampling columns: x_s (n*H*W, C) S32, off (n*H*W, >= 18) fp32 -> (groups, n*H*W, 9*C/groups) S32."""
    C = x_s.shape[-1]
    rows = n * H * W
    assert x_s.numel() == rows * C and off.dim() == 2 and off.shape[0] == rows
    cols = torch.empty((groups, rows, 9 * C // groups), dtype=torch.float32, device=x_s.device)
    _call("occ_deform_im2col", x_s, off, off.shape[1], cols, n, H, W, C, groups)
    return cols


def modulated_deform_im2col(x_s, off, n, H, W):
    """DCNv2 sampling columns: x_s (n*H*W, C) S32, off (n*H*W, >= 27) fp32 conv_offset rows (dy, dx of point k in columns
    2k, 2k+1, its mask logit in column 18 + k) -> (n*H*W, 9*C) S32, column k*C + c = sigmoid(logit_k) * sample."""
    C = x_s.shape[-1]
    rows = n * H * W
    assert x_s.numel() == rows * C and off.dim() == 2 and off.shape[0] == rows
    cols = torch.empty((rows, 9 * C), dtype=torch.float32, device=x_s.device)
    _call("occ_modulated_deform_im2col", x_s, off, off.shape[1], cols, n, H, W, C)
    return cols


# ----------------------------------------------------------------------------------------------- image encoder
STEM_COLS = 160  # the 147 (ky, kx, c) columns of the 7x7x3 stem, padded to whole S32 chunks


def split_nchw(x):
    """x (n, C, H, W) fp32 CUDA image map -> its S32 channel-last rows (n, H, W, C), C % 32 == 0.  A channels_last tensor
    (what this package's image encoder returns) is split in place order by occ_split_rows; any other layout goes through
    the transposing split of occ_head_prep."""
    n, C, H, W = x.shape
    if x.is_contiguous(memory_format=torch.channels_last):
        return to_split(x.permute(0, 2, 3, 1))
    return head_prep(x.contiguous().view(n, C, H * W), False)[0].view(n, H, W, C)


def stem_im2col(img):
    """img (n, 3, H, W) fp32 -> S32 columns (n*Ho*Wo, 160) of the 7x7 stride-2 pad-3 stem, column (ky*7 + kx)*3 + c,
    Ho = (H - 1)//2 + 1 (occ_stem_im2col)."""
    n, c, H, W = img.shape
    return im2col3(img, 7, 2, 3, 3, (H - 1) // 2 + 1, (W - 1) // 2 + 1, STEM_COLS)


def im2col3(img, k, stride, pad_top, pad_left, Ho, Wo, ncols):
    """img (n, 3, H, W) fp32 -> S32 columns (n*Ho*Wo, ncols) of a k x k conv on 3 channels: column (ky*k + kx)*3 + c =
    img[c, stride*oy - pad_top + ky, stride*ox - pad_left + kx], 0 outside the image and in columns >= 3*k*k
    (occ_stem_im2col)."""
    n, c, H, W = img.shape
    assert c == 3 and ncols % 32 == 0 and ncols >= 3 * k * k
    cols = torch.empty((n * Ho * Wo, ncols), dtype=torch.float32, device=img.device)
    _call("occ_stem_im2col", img, cols, n, H, W, k, stride, pad_top, pad_left, Ho, Wo, ncols)
    return cols


def maxpool3x3s2(x):
    """x (n, H, W, C) channel-last fp32 -> S32 (n, Ho, Wo, C): nn.MaxPool2d(3, 2, 1) (occ_maxpool3x3s2)."""
    n, H, W, C = x.shape
    out = torch.empty((n, (H - 1) // 2 + 1, (W - 1) // 2 + 1, C), dtype=torch.float32, device=x.device)
    _call("occ_maxpool3x3s2", x, out, n, H, W, C)
    return out


def space_to_depth(x, f):
    """x (n, H, W, C) -> (n, H/f, W/f, f*f*C), column (i*f + j)*C + c = x[f*y + i, f*x + j, c] (S32 stays S32)."""
    n, H, W, C = x.shape
    out = torch.empty((n, H // f, W // f, f * f * C), dtype=torch.float32, device=x.device)
    _call("occ_space_to_depth", x, out, n, H, W, C, f)
    return out


def depth_to_space_into(x, n, h, w, f, out, out_off):
    """x (n*h*w, f*f*C) fp32 -> columns [out_off, out_off + C) of out (n*f*h*f*w, ldo), row (b, f*y + i, f*x + j) from
    column (i*f + j)*C + c of row (b, y, x); the other columns are left as they are.  -> out"""
    C = x.shape[1] // (f * f)
    assert x.shape == (n * h * w, f * f * C) and out.dim() == 2 and out.shape[0] == n * h * w * f * f
    _call("occ_depth_to_space", x, out, n, h, w, C, f, out.shape[1], out_off)
    return out


# ----------------------------------------------------------------------------------------------- EfficientNet block
def dwconv_swish(x, w, b, k, stride, pad_top, pad_left, Ho, Wo):
    """Depthwise k x k conv + folded BatchNorm + Swish: x (n, H, W, C) fp32, w (k*k, C) tap-major, b (C) -> (out (n, Ho,
    Wo, C) fp32, SE partial sums (n, tiles, C)) (occ_dwconv_swish)."""
    n, H, W, C = x.shape
    tiles = lib().occ_dw_tiles(Ho, Wo)
    out = torch.empty((n, Ho, Wo, C), dtype=torch.float32, device=x.device)
    part = torch.empty((n, tiles, C), dtype=torch.float32, device=x.device)
    _call("occ_dwconv_swish", x, w, b, out, part, n, H, W, C, k, stride, pad_top, pad_left, Ho, Wo)
    return out, part


def se_gate(part, hw, w1T, b1, w2T, b2):
    """SELayer gate from occ_dwconv_swish's partial sums (n, tiles, C) of an hw-pixel map: w1T (C, S), b1 (S), w2T (S, C),
    b2 (C) -> gate (n, C) = sigmoid(W2 swish(W1 mean + b1) + b2) (occ_se_gate)."""
    n, tiles, C = part.shape
    S = b1.shape[0]
    gate = torch.empty((n, C), dtype=torch.float32, device=part.device)
    _call("occ_se_gate", part, tiles, hw, w1T, b1, w2T, b2, gate, n, C, S)
    return gate


def se_scale(y, gate):
    """y (n, ..., C) fp32, gate (n, C) -> y * gate[image] in S32, same shape (occ_se_scale)."""
    n, C = gate.shape
    out = torch.empty_like(y)
    _call("occ_se_scale", y, gate, out, n, y.numel() // (n * C), C)
    return out


# ----------------------------------------------------------------------------------------------- encoder glue
_WL = {}


def window_layout_buffer(B, X, Y, Z, C, shift, device):
    """Zero-initialised window-layout token buffer (occ_window_layout_rows, C), cached per (grid, shift, device, stream):
    the producer overwrites exactly the rows of real tokens on every call, the pad rows stay zero for ever."""
    key = (B, X, Y, Z, C, int(bool(shift)), str(device), torch.cuda.current_stream(device).cuda_stream)
    buf = _WL.get(key)
    if buf is None:
        rows = lib().occ_window_layout_rows(B, X, Y, Z)
        assert rows > 0
        buf = _WL[key] = torch.zeros((rows, C), dtype=torch.float32, device=device)
    return buf


def window_layout_index(B, X, Y, Z, shift):
    """Token row (voxel tokens, then BEV tokens) -> row of the window-layout buffer, as an int64 tensor (host arithmetic,
    independent of the kernels: tests and callers that hold token-ordered rows)."""
    WS = 7
    nWx, nWy = (X + WS - 1) // WS, (Y + WS - 1) // WS
    Xp, Yp = nWx * WS, nWy * WS
    x = torch.arange(X).view(X, 1)
    y = torch.arange(Y).view(1, Y)
    xs, ys = ((x - 3) % Xp, (y - 3) % Yp) if shift else (x, y)
    win_xy = (xs // WS) * nWy + (ys // WS)              # (X, Y)
    t = (xs % WS) * WS + (ys % WS)                      # (X, Y)
    b = torch.arange(B).view(B, 1, 1, 1)
    z = torch.arange(Z).view(1, 1, 1, Z)
    img = b * Z + z                                     # voxel slice image index
    nimg = B * (Z + 1)                                  # window index = (wx * nWy + wy) * n_images + image
    vox = (win_xy.view(1, X, Y, 1) * nimg + img) * 64 + t.view(1, X, Y, 1)                # (B, X, Y, Z)
    bev = (win_xy.view(1, X, Y) * nimg + (B * Z + torch.arange(B).view(B, 1, 1))) * 64 + t.view(1, X, Y)
    return torch.cat([vox.reshape(-1), bev.reshape(-1)]).long()


def to_window_layout(tokn_s, B, X, Y, Z, shift):
    """token-ordered (rows, C) rows -> window-layout buffer (fresh tensor)"""
    rows = lib().occ_window_layout_rows(B, X, Y, Z)
    out = torch.zeros((rows, tokn_s.shape[1]), dtype=tokn_s.dtype, device=tokn_s.device)
    out[window_layout_index(B, X, Y, Z, shift).to(tokn_s.device)] = tokn_s
    return out


def gn_relu_zmean_ln(y, stats, gn_w, gn_b, ln_w, ln_b, B, XY, Z, C, groups, X=0, win_shift=None):
    """-> tok (fp32, token order), tokn (S32): token order, or -- win_shift = 0 / 1 -- the window layout of that partition
    (operand of swin_qkv_attention)."""
    rows = B * XY * (Z + 1)
    tok = torch.empty((rows, C), dtype=torch.float32, device=y.device)
    if win_shift is None:
        tokn = torch.empty((rows, C), dtype=torch.float32, device=y.device)
        ws = -1
    else:
        assert X > 0 and XY % X == 0
        tokn = window_layout_buffer(B, X, XY // X, Z, C, win_shift, y.device)
        ws = int(bool(win_shift))
    _call("occ_gn_relu_zmean_ln", y, stats, gn_w, gn_b, ln_w, ln_b, tok, tokn, B, XY, Z, C, groups, X, ws)
    return tok, tokn


def layernorm(x, w, b, split_out=False):
    rows, C = x.shape
    out = torch.empty_like(x)
    _call("occ_layernorm", x, w, b, out, rows, C, int(split_out))
    return out


def swin_proj_ffn(att, tok, wp, bp, ln_w, ln_b, w1, b1, w2, b2):
    """Fused Swin block tail (C == 128): tok + proj(att) -> LN2 -> FFN(GELU) + residual, one kernel."""
    M, C = att.shape
    assert tok.shape == (M, C) and wp.shape == (C, C) and w1.shape == (C, C) and w2.shape == (C, C)
    out = torch.empty_like(att)
    _call("occ_swin_proj_ffn", att, tok, wp, bp, ln_w, ln_b, w1, b1, w2, b2, out, M, C)
    return out


def gn_apply(x, stats, w, b, rows_per_batch, groups, residual=None, relu=True, want_f32=True, split_into=None,
             out_off=0, want_split=False, out_f32=None):
    """GroupNorm apply (+ReLU, +residual) of a raw conv output x (rows, C).  Returns (out_f32 | None, out_s32 | None):
    the fp32 result when want_f32, the S32 result written into split_into[:, out_off:out_off+C] (or a fresh (rows, C)
    tensor when want_split)."""
    rows, C = x.shape
    out = out_f32 if out_f32 is not None else (torch.empty_like(x) if want_f32 else None)
    if out is not None:
        assert out.shape == x.shape
    if split_into is None and want_split:
        split_into = torch.empty_like(x)
    ldo = split_into.shape[1] if split_into is not None else C
    _call("occ_gn_apply", x, stats, w, b, residual, out, split_into, rows, rows_per_batch, C, groups, ldo, out_off,
          int(relu))
    return out, split_into


def aspp_gap_branch(x, wconv, gw, gb, cat, B, rows_per_batch, groups, out_off):
    ch = x.shape[1]
    sums = torch.empty((B, ch * 3 // 2 + 2), dtype=torch.float64, device=x.device)  # B*ch doubles + B*ch floats
    _call("occ_aspp_gap_branch", x, sums, wconv, gw, gb, cat, B, rows_per_batch, ch, groups, cat.shape[1], out_off)
    return cat


def dualpath_fuse(x, bev, cw, cbias, identity, B, XY, Z, C, identity_split=False, id_stats=None, id_w=None, id_b=None,
                  groups=0, want_f32=True, want_split=True):
    """-> (out fp32 | None, out S32 | None), each (B*XY*Z, C)."""
    out = torch.empty((B * XY * Z, C), dtype=torch.float32, device=x.device) if want_f32 else None
    out_s = torch.empty((B * XY * Z, C), dtype=torch.float32, device=x.device) if want_split else None
    _call("occ_dualpath_fuse", x, bev, cw, float(cbias), identity, int(identity_split), id_stats, id_w, id_b, groups,
          out, out_s, B, XY, Z, C)
    return out, out_s


def qkv_head_major_perm(C, heads, device=None):
    """row permutation of WindowMSA.qkv (weight / bias): new row h*96 + which*32 + d <- reference row which*C + h*32 + d."""
    hd = C // heads
    idx = torch.arange(3 * C, device=device).view(3, heads, hd).permute(1, 0, 2).reshape(-1)
    return idx


def window_attention(qkv, qkv_bias, bias_pad, B, X, Y, Z, C, heads, shift, head_major=False):
    rows = B * X * Y * (Z + 1)
    assert qkv.shape == (rows, 3 * C)
    out = torch.empty((rows, C), dtype=torch.float32, device=qkv.device)
    _call("occ_window_attention", qkv, qkv_bias, bias_pad, out, B, X, Y, Z, C, heads, int(shift), int(head_major))
    return out


def swin_qkv_attention(tokn_wl, w_qkv, b_qkv, bias_pad, B, X, Y, Z, C, heads, shift):
    """QKV projection + (shifted) window attention in one kernel (C == 128): tokn_wl (window_layout rows, C) S32 in the
    window layout of ``shift`` (gn_relu_zmean_ln(win_shift=shift) / to_window_layout), w_qkv (3C, C) S32 and b_qkv (3C,)
    fp32 with head-major rows -> attention output (B*X*Y*(Z+1), C) S32 in token order."""
    rows = B * X * Y * (Z + 1)
    assert tokn_wl.shape == (lib().occ_window_layout_rows(B, X, Y, Z), C) and w_qkv.shape == (3 * C, C)
    out = torch.empty((rows, C), dtype=torch.float32, device=tokn_wl.device)
    _call("occ_swin_qkv_attention", tokn_wl, w_qkv, b_qkv, bias_pad, out, B, X, Y, Z, C, heads, int(shift))
    return out


# ----------------------------------------------------------------------------------------------- decoder head
def sine_pos3d(X, Y, Z, num_feats, device, temperature=10000.0, scale=6.283185307179586, eps=1e-6, offset=0.0):
    out = torch.empty((X * Y * Z, 3 * num_feats), dtype=torch.float32, device=device)
    _call("occ_sine_pos3d", out, X, Y, Z, num_feats, temperature, scale, eps, offset)
    return out


def head_prep(x, channel_last, level_embed=None, pos=None):
    """x: (B,S,C) channel-last memory or (B,C,S) reference layout -> mem (B,S,C) [, kpos (B,S,C)] in S32."""
    if channel_last:
        B, S, C = x.shape
    else:
        B, C, S = x.shape
    mem = torch.empty((B, S, C), dtype=torch.float32, device=x.device)
    kpos = torch.empty_like(mem) if pos is not None else None
    _call("occ_head_prep", x, int(channel_last), level_embed, pos, mem, kpos, B, S, C)
    return mem, kpos


def query_head(query_in, W, NC, norm2=None, next_q=None, ffn_part=None):
    """forward_head query side.  norm2 = (w, b): query_in is the FFN accumulator, LN(norms.2) gives the layer output
    (returned as `query`); next_q = (query_pos, Q, wqT, bq, scale): also project the next layer's cross-attn queries."""
    rows, E = query_in.shape
    cls = torch.empty((rows, NC), dtype=torch.float32, device=query_in.device)
    membed = torch.empty((rows, E), dtype=torch.float32, device=query_in.device)
    query = torch.empty_like(query_in) if norm2 is not None else query_in
    qh = torch.empty_like(query_in) if next_q is not None else None
    n2w, n2b = norm2 if norm2 is not None else (None, None)
    qpos, Q, wqT, bq, scale = next_q if next_q is not None else (None, 0, None, None, 0.0)
    _call("occ_query_head", query_in, n2w, n2b, query if norm2 is not None else None, W["pn_w"], W["pn_b"], W["clsT"],
          W["cls_b"], NC, W["m0T"], W["m0b"], W["m1T"], W["m1b"], W["m2T"], W["m2b"], cls, membed, qpos, Q, wqT, bq,
          scale, qh, ffn_part, ffn_part.shape[0] if ffn_part is not None else 0, rows, E)
    return cls, membed, query, qh


def decode_ordered(t):
    """order-preserving int32 -> float32 (inverse of the kernels' encoding; used by tests / debugging)."""
    i = t.to(torch.int32)
    return torch.where(i >= 0, i, i ^ 0x7FFFFFFF).view(torch.float32)


def mask_pool(mask, B, grid, out_grid, Q):
    """General adaptive max pool of the query-last mask logits -> (pooled ordered-int32 (B,So,Q), flag int32 (B*Q,))."""
    X, Y, Z = grid
    Xo, Yo, Zo = out_grid
    pooled = torch.empty((B, Xo * Yo * Zo, Q), dtype=torch.int32, device=mask.device)
    flag = torch.empty((B * Q,), dtype=torch.int32, device=mask.device)
    _call("occ_mask_pool", mask, pooled, flag, B, X, Y, Z, Xo, Yo, Zo, Q)
    return pooled, flag


def mask_gemm_pool(mf_r, membed, B, grid, out_grid, Q):
    """Pooled attention-mask logits straight from the mask features, without the (B,V,Q) logits: -> (pooled, flag) as
    mask_pool, or None for a shape the kernel does not cover (nothing was launched: compute the logits with gemm and pool
    them with mask_pool)."""
    X, Y, Z = grid
    Xo, Yo, Zo = out_grid
    E = mf_r.shape[-1]
    pooled = torch.empty((B, Xo * Yo * Zo, Q), dtype=torch.int32, device=mf_r.device)
    flag = torch.empty((B * Q,), dtype=torch.int32, device=mf_r.device)
    if _call("occ_mask_gemm_pool", mf_r, membed, pooled, flag, B, X, Y, Z, E, Q, Xo, Yo, Zo, unsupported_ok=True) == -2:
        return None
    return pooled, flag


def cross_attn_tc(qh, Kp, Vp, ld, koff, voff, pooled, flag, B, S, Q, E, H):
    """Masked cross attention on the tensor cores -> (partials (B,H,npart,Q,34), npart)."""
    npart = lib().occ_cross_attn_tc_partials(S)
    part = torch.empty((B, H, npart, Q, 34), dtype=torch.float32, device=qh.device)
    bits = torch.empty((B, 4 * ((S + 127) // 128), Q), dtype=torch.int32, device=qh.device)
    _call("occ_mask_bits", pooled, bits, B, S, Q)
    _call("occ_cross_attn_tc", qh, Kp, Vp, ld, koff, voff, bits, flag, part, B, S, Q, E, H)
    return part, npart


def cross_merge(part, nchunk, H, query, query_pos, Q, L, scale):
    rows, E = query.shape
    q1 = torch.empty_like(query)
    sa = torch.empty((rows, 3 * E), dtype=torch.float32, device=query.device)
    _call("occ_cross_merge", part, nchunk, H, query, query_pos, Q, L["ca_woT"], L["ca_bo"], L["n0w"], L["n0b"],
          L["sa_inT"], L["sa_inb"], scale, q1, sa, rows, E)
    return q1, sa


def self_attn_ffn(sa, q1, Q, L, H, nkeys=None):
    """-> (ybuf = x1 + b2, ffn_part (F/E, rows, E)): the pre-norms.2 accumulator of the decoder layer and the FFN
    column-block partials that occ_query_head adds to it in a fixed order.  Q query slots per sample, of which the first
    nkeys (default Q) are the self-attention keys."""
    rows, E = q1.shape
    x1 = torch.empty_like(q1)
    ybuf = torch.empty_like(q1)
    F = L["f1b"].numel()
    part = torch.empty((F // E, rows, E), dtype=torch.float32, device=q1.device)
    _call("occ_self_attn_ffn", sa, q1, Q, Q if nkeys is None else nkeys, L["sa_woT"], L["sa_bo"], L["n1w"], L["n1b"],
          L["f1T"], L["f1b"], L["f2T"], L["f2b"], F, x1, ybuf, part, rows, E, H)
    return ybuf, part


def classmix(mask, cls, B, grid, out_grid, Q, NC, with_labels=False):
    """mask (B, S, Qs) query-last logits with Qs >= Q slots per row, cls (B, Q, NC) -> class volume (B, NC-1, *out_grid)
    [, uint8 labels]."""
    X, Y, Z = grid
    Xo, Yo, Zo = out_grid
    out = torch.empty((B, NC - 1, Xo, Yo, Zo), dtype=torch.float32, device=mask.device)
    labels = torch.empty((B, Xo, Yo, Zo), dtype=torch.uint8, device=mask.device) if with_labels else None
    _call("occ_classmix", mask, mask.shape[-1], cls, out, labels, B, X, Y, Z, Xo, Yo, Zo, Q, NC)
    return (out, labels) if with_labels else out


def thing_mask(thing_indices):
    """class indices -> the bit mask of occ_panoptic_voxels / occ_panoptic_points"""
    m = 0
    for k in thing_indices or ():
        assert 0 <= int(k) < 64, f"thing class index {k} out of range"
        m |= 1 << int(k)
    return m


def _panoptic_ws(B, n, Qs, device):
    return (torch.empty((B, n), dtype=torch.uint8, device=device), torch.empty((B, Qs), dtype=torch.int32, device=device),
            torch.empty((B, Qs, 2), dtype=torch.int64, device=device))


def panoptic_voxels(mask, cls, B, grid, out_grid, Q, thing, point_rule=False):
    """mask (B, S, Qs) query-last logits, cls (B, Q, NC), thing = thing_mask(...) -> (semantic, panoptic) int64
    (B, *out_grid): format_panoptic_occupancy_results of the trilinearly upsampled logits; point_rule: the label rule of
    format_panoptic_lidar_results (class 0 is never a label)."""
    X, Y, Z = grid
    Xo, Yo, Zo = out_grid
    Qs, NC = mask.shape[-1], cls.shape[-1]
    assert cls.shape == (B, Q, NC) and mask.shape == (B, X * Y * Z, Qs)
    sem = torch.empty((B, Xo, Yo, Zo), dtype=torch.int64, device=mask.device)
    pan = torch.empty_like(sem)
    qidx, present, table = _panoptic_ws(B, Xo * Yo * Zo, Qs, mask.device)
    _call("occ_panoptic_voxels", mask, Qs, cls, B, X, Y, Z, Xo, Yo, Zo, Q, NC, thing, int(point_rule), qidx, present,
          table, sem, pan)
    return sem, pan


def panoptic_points(mask, cls, B, grid, Q, thing, pts, pc_range, border=True):
    """mask (B, S, Qs) native query-last logits, cls (B, Q, NC), pts (B, n, >=3) -> (semantic, panoptic) int64 (B, n):
    forward_lidar_panopticseg, eval branch."""
    X, Y, Z = grid
    Qs, NC = mask.shape[-1], cls.shape[-1]
    assert cls.shape == (B, Q, NC) and mask.shape == (B, X * Y * Z, Qs)
    pts = pts.to(mask.device).float().contiguous()
    assert pts.dim() == 3 and pts.shape[0] == B and pts.shape[2] >= 3
    n = pts.shape[1]
    sem = torch.zeros((B, n), dtype=torch.int64, device=mask.device)
    pan = torch.zeros_like(sem)
    qidx, present, table = _panoptic_ws(B, n, Qs, mask.device)
    r = [float(v) for v in pc_range]
    _call("occ_panoptic_points", mask, Qs, cls, B, X, Y, Z, Q, NC, thing, pts, pts.shape[2], n, *r, int(border), qidx,
          present, table, sem, pan)
    return sem, pan


def transpose_sq(mask, B, S, Q):
    out = torch.empty((B, Q, S), dtype=torch.float32, device=mask.device)
    _call("occ_transpose_sq", mask, out, B, S, Q)
    return out


def lidarseg_points(vox, pts, pc_range, border=True):
    """vox (K,X,Y,Z) contiguous class volume of one sample; pts (n, >=3) -> (n, K) softmaxed point scores."""
    K, X, Y, Z = vox.shape
    pts = pts.float().contiguous()
    n = pts.shape[0]
    out = torch.empty((n, K), dtype=torch.float32, device=vox.device)
    r = [float(v) for v in pc_range]
    _call("occ_lidarseg_points", vox, pts if n else None, pts.shape[1] if n else 3, n, r[0], r[1], r[2], r[3], r[4],
          r[5], X, Y, Z, K, int(border), out)
    return out


# ----------------------------------------------------------------------------------------------- neck (pixel decoder)
def _grids_arr(grids):
    flat = [int(v) for g in grids for v in g]
    return (ctypes.c_int * len(flat))(*flat)


def gn_stats(x, B, rows_per_batch, C, groups):
    """fp64 (sum, sumsq) per (sample, group) of a finished tensor x (B*rows_per_batch, C), C % 4 == 0, at most 96 groups
    -> (B, groups, 2); for a conv whose bias comes before the GroupNorm (the epilogue statistics are of the raw output)."""
    stats = torch.zeros((B, groups, 2), dtype=torch.float64, device=x.device)
    _call("occ_gn_stats", x, stats, B, rows_per_batch, C, C // groups)
    return stats


def neck_token_prep(x, grids, B, ln=None, pos=None, want_f32=True, want_s32=True, want_pos=False):
    """[LayerNorm] of level-major token rows x (B*Nq, C) -> (x fp32 | None, x S32 | None, (x + pos) S32 | None)."""
    rows, C = x.shape
    f32 = torch.empty_like(x) if want_f32 else None
    s32 = torch.empty_like(x) if want_s32 else None
    ps = torch.empty_like(x) if want_pos else None
    lw, lb = ln if ln is not None else (None, None)
    _call("occ_neck_token_prep", x, lw, lb, pos, f32, s32, ps, len(grids), B, _grids_arr(grids), C)
    return f32, s32, ps


def neck_layer_tail(att, x, wo, bo, ln1, w1, b1, w2, b2, ln2, grids, B, pos=None, want_f32=True, want_s32=True,
                    want_pos=False):
    """One pixel-decoder encoder layer after the deformable gather, one kernel: y = x + att wo^T + bo, x1 = LN1(y),
    out = LN2(x1 + w2 ReLU(w1 x1 + b1) + b2) -> (out fp32 | None, out S32 | None, (out + pos) S32 | None), the outputs of
    neck_token_prep.  att (rows, E) and the weights ((out, in) as in nn.Linear) in S32; ln1 / ln2 = (weight, bias)."""
    rows, E = x.shape
    F = w1.shape[0]
    assert att.shape == (rows, E) and wo.shape == (E, E) and w1.shape == (F, E) and w2.shape == (E, F)
    assert bo.shape == (E,) and b1.shape == (F,) and b2.shape == (E,)
    assert all(t.shape == (E,) for t in (*ln1, *ln2))
    assert rows == B * sum(gx * gy * gz for gx, gy, gz in grids) and (pos is not None or not want_pos)
    f32 = torch.empty_like(x) if want_f32 else None
    s32 = torch.empty_like(x) if want_s32 else None
    ps = torch.empty_like(x) if want_pos else None
    _call("occ_neck_layer_tail", att, x, wo, bo, ln1[0], ln1[1], w1, b1, w2, b2, ln2[0], ln2[1],
          pos if want_pos else None, f32, s32, ps, len(grids), B, _grids_arr(grids), E, F)
    return f32, s32, ps


def ms_deform_attn(value, ow, grids, strides, B, E, H, P):
    """3-D multi-scale deformable attention core on level-major rows -> (rows, E) in S32.  value (rows, H * head_ld): head h
    in columns [h*head_ld, h*head_ld + E/H) -- head_ld = E/H, or E/H rounded up to 32 (``pad_head_rows``)."""
    assert value.shape[1] % H == 0 and value.shape[1] // H >= E // H
    out = torch.empty(value.shape[0], E, dtype=torch.float32, device=value.device)
    st = (ctypes.c_float * len(strides))(*[float(v) for v in strides])
    _call("occ_ms_deform_attn", value, value.shape[1], value.shape[1] // H, ow, out, len(grids), B, _grids_arr(grids),
          st, E, H, P)
    return out


def pad_head_rows(w, b, H):
    """value_proj (E, K) weight / (E,) bias -> (H * hp, K) / (H * hp,) with hp = E/H rounded up to 32 and zero rows in the
    pad: the projection then writes every head slice into its own 128-byte line (see occ_ms_deform_attn)."""
    E = w.shape[0]
    hd = E // H
    hp = (hd + 31) // 32 * 32
    if hp == hd:
        return w.detach().float().contiguous(), b.detach().float().contiguous()
    wp = torch.zeros(H, hp, w.shape[1], dtype=torch.float32, device=w.device)
    wp[:, :hd] = w.detach().float().view(H, hd, -1)
    bp = torch.zeros(H, hp, dtype=torch.float32, device=w.device)
    bp[:, :hd] = b.detach().float().view(H, hd)
    return wp.view(H * hp, -1).contiguous(), bp.view(-1).contiguous()


def gn_upsample_add(cur, stats, gw, gb, groups, coarse):
    """cur (B,X,Y,Z,C) raw conv output (+ stats), coarse (B,Xc,Yc,Zc,C) fp32 -> GN(cur) + trilinear_up(coarse) in S32."""
    B, X, Y, Z, C = cur.shape
    _, Xc, Yc, Zc, _ = coarse.shape
    out = torch.empty_like(cur)
    _call("occ_gn_upsample_add", cur, stats, gw, gb, groups, coarse, out, B, X, Y, Z, Xc, Yc, Zc, C)
    return out


# ----------------------------------------------------------------------------------------------- evaluation tail
def ssc_counts(pred, target, K, ignore=255):
    """uint8 label volumes (any shape) -> int64 (3 + 3K,): completion tp/fp/fn, semantic tp/fp/fn per class."""
    p = pred.reshape(-1).to(torch.uint8).contiguous()
    t = target.reshape(-1).to(torch.uint8).contiguous()
    assert p.numel() == t.numel()
    ws = torch.empty(K * K, dtype=torch.int64, device=p.device)
    out = torch.empty(3 + 3 * K, dtype=torch.int64, device=p.device)
    _call("occ_ssc_counts", p, t, p.numel(), K, ignore, ws, out)
    return out


def _flat_ids(t, name):
    """integer (or whole-number floating) tensor of any shape -> flat contiguous int64"""
    if t.dtype == torch.bool or t.is_complex():
        raise RuntimeError(f"occformer_b200: {name} must hold integer ids, got {t.dtype}")
    return t.reshape(-1).to(torch.int64).contiguous()


def panoptic_eval(x_sem, x_inst, y_sem, y_inst, K, ignore_mask, min_points, state, parts=3):
    """PanopticEval.addBatch on one flat scan (occ_panoptic_eval): x = prediction, y = target, any shape and integer
    dtype; state: int64 (K*K + 6K + 1,) CUDA vector, accumulated in place.  parts: 1 = confusion matrix only, 2 = panoptic
    counts only, 3 = both.  -> state"""
    xs, ys = _flat_ids(x_sem, "x_sem"), _flat_ids(y_sem, "y_sem")
    xi = _flat_ids(x_inst, "x_inst") if parts & 2 else None
    yi = _flat_ids(y_inst, "y_inst") if parts & 2 else None
    n = xs.numel()
    if any(t is not None and t.numel() != n for t in (ys, xi, yi)):
        raise RuntimeError("occformer_b200: panoptic_eval inputs must have the same number of elements")
    assert state.numel() == K * K + 6 * K + 1, "panoptic state vector has the wrong length"
    nbytes = lib().occ_panoptic_eval_workspace_bytes(n)
    if nbytes == 0:
        raise RuntimeError(f"occformer_b200: panoptic evaluation of {n} elements exceeds the 2^29-element limit of one call")
    ws = _stream_workspace("occ_panoptic_eval", xs.device, nbytes)  # zeroed by every call
    _call("occ_panoptic_eval", xs, xi, ys, yi, n, K, ignore_mask, min_points, parts, ws, ws.numel(), state)
    return state


def lidarseg_hist(scores, labels, K, hist=None):
    labels = labels.long().contiguous()
    if hist is None:
        hist = torch.zeros((K - 1, K - 1), dtype=torch.int64, device=scores.device)
    _call("occ_lidarseg_hist", scores, labels, scores.shape[0], K, hist)
    return hist


# ----------------------------------------------------------------------------------------------- occupancy ground truth
def lidarseg_occupancy(pts, counts, pc_range, grid, panoptic, empty_id, ignore):
    """Occupancy ground truth of B samples (occ_lidarseg_occupancy): pts (n, ld >= 4) fp32 CUDA rows [x, y, z, label, ...],
    sample b the next counts[b] rows -> (int64 (B, X, Y, Z) volume, int32 (1,) invalid-point counter); no synchronisation."""
    B = len(counts)
    n, ld = pts.shape
    offsets = [0]
    for c in counts:
        offsets.append(offsets[-1] + int(c))
    assert offsets[-1] == n
    X, Y, Z = (int(v) for v in grid)
    dev = pts.device
    nbytes = lib().occ_lidarseg_occupancy_workspace_bytes(n, B)
    if nbytes == 0:
        raise RuntimeError(f"occformer_b200: occ_lidarseg_occupancy takes 1..256 samples and at most 2^30 points, "
                           f"got {B} samples, {n} points")
    ws = _stream_workspace("occ_lidarseg_occupancy", dev, nbytes)
    out = torch.empty((B, X, Y, Z), dtype=torch.int64, device=dev)
    invalid = torch.zeros(1, dtype=torch.int32, device=dev)
    r = [float(v) for v in pc_range]
    _call("occ_lidarseg_occupancy", pts, ld, (ctypes.c_longlong * (B + 1))(*offsets), B, *r, X, Y, Z, int(panoptic),
          int(empty_id), int(ignore), invalid, ws, ws.numel(), out)
    return out, invalid


def semkitti_labels(label, invalid, B, nvox, lut):
    """SemanticKITTI ground truth of B samples (occ_semkitti_labels): label uint8 CUDA (B * 2 * nvox,) bytes of the
    .label files, invalid uint8 CUDA (B * nvox / 8,) bytes of the .invalid files, lut int32 CUDA remap table ->
    (int64 (B, nvox) volume, int32 (B,) count of labels past the LUT per sample); no synchronisation."""
    out = torch.empty((B, nvox), dtype=torch.int64, device=label.device)
    bad = torch.zeros(B, dtype=torch.int32, device=label.device)
    _call("occ_semkitti_labels", label, invalid, B, nvox, lut, lut.numel(), bad, out)
    return out, bad


def semkitti_labels_aug(label, invalid, B, aug, lut):
    """the training-mode SemanticKITTI ground truth of B samples (occ_semkitti_labels_aug): label / invalid / lut as
    semkitti_labels with nvox = 256 * 256 * 32, aug int32 CUDA (B, 10) rows (flip_dx, flip_dy, flip_dz, rotate,
    a0..a5) -> (int64 (B, 256, 256, 32) volume, int32 (B,) count of labels past the LUT per sample); no
    synchronisation."""
    if label.numel() != B * 2 * 256 * 256 * 32 or invalid.numel() != B * 256 * 256 * 4 or aug.numel() != B * 10:
        raise RuntimeError(f"occformer_b200: occ_semkitti_labels_aug: B = {B} needs {B * 2 << 21} label bytes, "
                           f"{B << 18} invalid bytes and {B * 10} aug values, got {label.numel()}, {invalid.numel()}, "
                           f"{aug.numel()}")
    out = torch.empty((B, 256, 256, 32), dtype=torch.int64, device=label.device)
    bad = torch.zeros(B, dtype=torch.int32, device=label.device)
    _call("occ_semkitti_labels_aug", label, invalid, B, aug, lut, lut.numel(), bad, out)
    return out, bad


# ----------------------------------------------------------------------------------------------- camera images
def _image_prep():
    from . import image_prep  # image_prep imports ops at its top, so ops imports image_prep at call time
    return image_prep


def _prep_table(dev, in_size, out_size):
    """the int32 resample table of one axis (image_prep.resample_table) on dev"""
    return _device_table(dev, ("resample", in_size, out_size),
                         lambda: _image_prep().resample_table(in_size, out_size))


def prepare_images(frames, offsets, geoms, input_size, mean, std, to_rgb, aug=None):
    """M camera images from uint8 BGR frames (occ_prepare_images): frames a flat uint8 CUDA buffer, image m the H x W x 3
    bytes at offsets[m], geoms[m] = (H, W, rW, rH, x0, y0) -> float32 (M, 3, fH, fW).  aug: None, or per image
    (flip, a0, .., a5), the training loaders' flip and rotation (occ_prepare_images_aug).  The coefficient and
    normalisation tables are built once per geometry and config and kept on the device; no synchronisation."""
    M = len(geoms)
    fH, fW = (int(v) for v in input_size)
    dev = frames.device
    geom = (ctypes.c_int * (6 * M))(*[int(v) for g in geoms for v in g])
    norm = _device_table(dev, ("normalize", tuple(mean), tuple(std), bool(to_rgb)),
                         lambda: _image_prep().normalize_table(mean, std, to_rgb))
    tables = []
    for H, W, rW, rH, _, _ in geoms:
        tables += [_prep_table(dev, W, rW).data_ptr(), _prep_table(dev, H, rH).data_ptr()]
    nbytes = lib().occ_prepare_images_workspace_bytes(geom, M, fH, fW)
    ws = _stream_workspace("occ_prepare_images", dev, max(nbytes, 16))
    out = torch.empty((M, 3, fH, fW), dtype=torch.float32, device=dev)
    head = [frames, frames.numel(), (ctypes.c_longlong * M)(*offsets), geom]
    tail = [M, fH, fW, (ctypes.c_longlong * (2 * M))(*tables), norm, int(bool(to_rgb)), ws, ws.numel(), out]
    if aug is None:
        _call("occ_prepare_images", *head, *tail)
    else:
        _call("occ_prepare_images_aug", *head, (ctypes.c_int * (7 * M))(*[int(v) for a in aug for v in a]), *tail)
    return out


def lidar_depth(pts, offsets, inv_rots, trans, intrins, post_rots, post_trans, input_size):
    """Depth maps of B samples x N cameras (occ_lidar_depth): pts (n, 3) fp32 CUDA, sample b's points at rows
    [offsets[b], offsets[b + 1]); inv_rots, trans, intrins (3 x 3 or 4 x 4), post_rots, post_trans fp32 CUDA (B, N, ...)
    -> float32 (B, N, fH, fW); no synchronisation."""
    B, N = trans.shape[:2]
    fH, fW = (int(v) for v in input_size)
    out = torch.empty((B, N, fH, fW), dtype=torch.float32, device=trans.device)
    _call("occ_lidar_depth", pts if pts.numel() else None, (ctypes.c_longlong * (B + 1))(*offsets), B, N, inv_rots,
          trans, intrins, int(intrins.shape[-1]), post_rots, post_trans, fH, fW, out)
    return out


# ----------------------------------------------------------------------------------------------- JPEG decoding
JPEG_SEQ_BITS = 4096    # bits per subsequence of the parallel Huffman decode (scripts/bench_jpeg.py --tune)
JPEG_SYNC_ROUNDS = 6    # self-synchronisation rounds before the serial fix-up
JPEG_MAX_IMAGES = 96    # images per occ_decode_jpeg call


def _jpeg_table(dev, key, table):
    """a DQT / DHT table of jpeg.parse (key: its marker bytes, table: int32 numpy) on dev"""
    return _device_table(dev, key, lambda: table)


def decode_jpeg(data, offsets, headers, seq_bits=JPEG_SEQ_BITS, sync_rounds=JPEG_SYNC_ROUNDS):
    """M baseline JPEG files -> uint8 B, G, R frames (occ_decode_jpeg): data a flat uint8 CUDA buffer, file m at byte
    offsets[m], headers[m] = occformer_b200.jpeg.parse of it -> (out: flat uint8 CUDA buffer of the M (H, W, 3) frames
    back to back, status: int32 CUDA (M, 2), see include/occ_b200.h).  The Huffman and quantisation tables are uploaded
    once per distinct marker content and kept on the device; no synchronisation."""
    M = len(headers)
    if not 1 <= M <= JPEG_MAX_IMAGES:
        raise ValueError(f"decode_jpeg: 1 to {JPEG_MAX_IMAGES} images per call, got {M}")
    dev = data.device
    scan, geom, tables, out_off, total = [], [], [], [], 0
    for off, h in zip(offsets, headers):
        scan += [int(off) + h.scan_off, h.scan_len]
        geom += [h.height, h.width, h.hs, h.vs, h.restart]
        tables += [_jpeg_table(dev, *t).data_ptr() for t in h.qt + h.dc + h.ac]
        out_off.append(total)
        total += h.height * h.width * 3
    scan = (ctypes.c_longlong * (2 * M))(*scan)
    geom = (ctypes.c_int * (5 * M))(*geom)
    nbytes = lib().occ_decode_jpeg_workspace_bytes(scan, geom, M, int(seq_bits))
    if nbytes == 0:
        raise RuntimeError(f"occformer_b200: occ_decode_jpeg takes 32 <= seq_bits <= 2^20, got {seq_bits}")
    ws = _stream_workspace("occ_decode_jpeg", dev, nbytes)
    out = torch.empty(max(total, 1), dtype=torch.uint8, device=dev)
    status = torch.empty((M, 2), dtype=torch.int32, device=dev)
    _call("occ_decode_jpeg", data, data.numel(), scan, geom, (ctypes.c_longlong * (9 * M))(*tables),
          (ctypes.c_longlong * M)(*out_off), M, int(seq_bits), int(sync_rounds), ws, ws.numel(), out, out.numel(),
          status)
    return out[:total], status


# ----------------------------------------------------------------------------------------------- PNG decoding
PNG_MAX_IMAGES = 96     # images per occ_decode_png call
PNG_LAUNCHES = 37       # enqueued launches and memsets per call (include/occ_b200.h)


def decode_png(data, offsets, headers, idat):
    """M 8-bit RGB PNG files -> uint8 B, G, R frames (occ_decode_png): data a flat uint8 CUDA buffer holding image m's
    zlib stream at byte offsets[m], headers[m] = occformer_b200.png.parse of the file, idat an int32 CUDA tensor of
    every image's IDAT chunk starts in its stream (in image order) -> (out: flat uint8 CUDA buffer of the M (H, W, 3)
    frames back to back, status: int32 CUDA (M, 2), see include/occ_b200.h).  No synchronisation."""
    M = len(headers)
    if not 1 <= M <= PNG_MAX_IMAGES:
        raise ValueError(f"decode_png: 1 to {PNG_MAX_IMAGES} images per call, got {M}")
    dev = data.device
    geom, out_off, total = [], [], 0
    for h in headers:
        geom += [h.height, h.width, h.stream_len, h.cinfo]
        out_off.append(total)
        total += h.height * h.width * 3
    streams = (ctypes.c_longlong * M)(*[int(o) for o in offsets])
    geom = (ctypes.c_int * (4 * M))(*geom)
    counts = (ctypes.c_int * M)(*[len(h.idat) for h in headers])
    nbytes = lib().occ_decode_png_workspace_bytes(streams, geom, counts, M)
    if nbytes == 0:
        raise RuntimeError("occformer_b200: occ_decode_png refused the geometry or the streams")
    ws = _stream_workspace("occ_decode_png", dev, nbytes)
    out = torch.empty(max(total, 1), dtype=torch.uint8, device=dev)
    status = torch.empty((M, 2), dtype=torch.int32, device=dev)
    _call("occ_decode_png", data, data.numel(), streams, geom, counts, idat, idat.numel(),
          (ctypes.c_longlong * M)(*out_off), M, ws, ws.numel(), out, out.numel(), status)
    return out[:total], status
