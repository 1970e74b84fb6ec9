"""The conventions every module of this package that runs on the kernels shares: the prepared-parameter cache, the eval
BatchNorm fold, and the S32-twin hand-off between modules (DESIGN.md section 1)."""
import torch
import torch.nn as nn

_BN_TYPES = ("BN", "BN2d", "SyncBN", "NaiveSyncBN")  # identical in eval mode


def round32(c):
    return (c + 31) // 32 * 32


def _drop_prepared(module, incompatible_keys):
    module._prep = None


class PreparedModule(nn.Module):
    """A module whose CUDA forward reads its parameters in the kernels' layouts.  ``prepared()`` is the result of
    ``_prepare()`` (a pure function of the parameters and buffers), computed on first use and kept until load_state_dict
    or .to() / .cuda() / .double() drops it.  In-place edits of parameters are not seen: change weights with one of
    those."""

    def __init__(self):
        super().__init__()
        self._prep = None
        self.register_load_state_dict_post_hook(_drop_prepared)

    def _apply(self, fn, *a, **k):
        self._prep = None
        return super()._apply(fn, *a, **k)

    def prepared(self):
        if self._prep is None:
            self._prep = self._prepare()
        return self._prep


def batchnorm(norm_cfg, channels, eps_default):
    """the BatchNorm2d an mmcv ``norm_cfg`` builds; NotImplementedError naming the type for any other norm"""
    cfg = dict(norm_cfg or {})
    kind = cfg.pop("type", "BN")
    if kind not in _BN_TYPES:
        raise NotImplementedError(f"occformer_b200: norm_cfg type {kind!r} is not supported (BatchNorm only)")
    cfg.pop("requires_grad", None)
    return nn.BatchNorm2d(channels, eps=cfg.get("eps", eps_default), momentum=cfg.get("momentum", 0.1))


@torch.no_grad()
def fold_bn(w, b, bn, out_dim=0):
    """eval BatchNorm folded into the layer before it, in fp64, rounded to fp32: w' = w * g / sqrt(var + eps) along the
    output dimension out_dim, b' = (b - mean) * g / sqrt(var + eps) + beta"""
    s = bn.weight.double() / torch.sqrt(bn.running_var.double() + bn.eps)
    b0 = b.double() if b is not None else torch.zeros_like(s)
    shape = [1] * w.dim()
    shape[out_dim] = -1
    wf = (w.double() * s.view(shape)).float().contiguous()
    return wf, ((b0 - bn.running_mean.double()) * s + bn.bias.double()).float().contiguous()


# A module hands its output on as an fp32 (n, C, *spatial) view of channel-last memory that carries the S32 (split-bf16)
# copy the producer wrote anyway, so that the next module of this package need not split it again.
def attach_twin(view, s32):
    """Attach s32, the S32 copy of view in the layout (n, *spatial, round32(C)) (pad columns zero), to view and stamp it
    with view's version counter.  -> view"""
    view._occ_s32 = s32
    view._occ_s32_version = None if view.is_inference() else view._version
    return view


def twin_of(t):
    """The S32 twin attach_twin gave t while it still holds t's values, else None: None when t changed in place since
    (an in-place op on t, on its base or on another view of it moves the version counter they share), when the twin
    was not attached by attach_twin, or when it is not fp32 (n, *spatial, round32(C)) on t's device.  An inference
    tensor has no version counter, so an in-place change to one is not detected."""
    s32 = getattr(t, "_occ_s32", None)
    if s32 is None or not hasattr(t, "_occ_s32_version"):
        return None
    if t._occ_s32_version != (None if t.is_inference() else t._version):
        return None
    if s32.dtype != torch.float32 or s32.device != t.device or \
            tuple(s32.shape) != (t.shape[0], *t.shape[2:], round32(t.shape[1])):
        return None
    return s32
