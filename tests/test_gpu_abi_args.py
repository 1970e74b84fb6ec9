"""GPU twin of test_cpu_abi_args: CUDA tensors of the wrong dtype, layout or device are rejected against the header's
pointer declarations while the recording fake stands in for the library; the real library enqueues nothing."""
import pytest
import torch

from util import FakeLibrary

pytestmark = pytest.mark.gpu


@pytest.fixture
def fake(monkeypatch):
    from occformer_b200 import ops
    f = FakeLibrary()
    monkeypatch.setattr(ops, "lib", lambda: f)
    return f


def _rejects(fake, match, call):
    from occformer_b200 import _lib
    n0 = _lib.lib().occ_launch_count()
    with pytest.raises(RuntimeError, match=match):
        call()
    torch.cuda.synchronize()
    assert fake.calls == [] and _lib.lib().occ_launch_count() == n0


def test_wrong_dtype_layout_or_placement_is_rejected(cuda, fake):
    from occformer_b200 import ops
    a, w = torch.zeros(8, 32, device=cuda), torch.zeros(16, 32, device=cuda)
    _rejects(fake, r"occ_gemm_bf16x3\(A\) must be torch.float32, got torch.float64", lambda: ops.gemm(a.double(), w))
    _rejects(fake, r"occ_mask_bits\(pooled\) must be torch.int32, got torch.int64",
             lambda: ops._call("occ_mask_bits", torch.zeros(1, 8, 4, dtype=torch.int64, device=cuda),
                               torch.zeros(1, 4, 4, dtype=torch.int32, device=cuda), 1, 8, 4))
    _rejects(fake, r"occ_layernorm\(in\) must be contiguous",
             lambda: ops.layernorm(torch.zeros(32, 8, device=cuda).t(), a[0], a[0]))
    # a module parameter left on the host next to CUDA activations
    _rejects(fake, r"occ_layernorm\(w\) must be a CUDA tensor", lambda: ops.layernorm(a, torch.zeros(32), a[0]))


def test_tensor_on_another_device_is_rejected(cuda, fake):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    from occformer_b200 import ops
    with torch.cuda.device(0):
        _rejects(fake, r"occ_split_rows\(in\) lives on cuda:1", lambda: ops.to_split(torch.zeros(4, 32, device="cuda:1")))


def test_valid_arguments_reach_the_library(cuda, fake, monkeypatch):
    """checked calls pass: plain tensors as their device pointers, and the camera-strided planes of lift_splat_fused (a
    channel slice of DepthNet's output) without a copy"""
    from occformer_b200 import ops
    monkeypatch.setattr(ops, "_ws_cache", {})  # the fake sizes the pooling workspace at 0 bytes
    a, w = torch.zeros(8, 32, device=cuda), torch.zeros(16, 32, device=cuda)
    out = ops.gemm(a, w)
    assert fake.calls == [("occ_gemm_bf16x3", (a.data_ptr(), w.data_ptr(), out.data_ptr(), 8, 16, 32, None, None, 0, 0,
                                               torch.cuda.current_stream().cuda_stream))]
    fake.calls.clear()
    z = lambda *s: torch.zeros(*s, device=cuda)  # noqa: E731
    y = z(2, 24, 3, 4)  # (B*N, D + C, fH, fW) with D = 8, C = 16
    ops.lift_splat_fused(y[:, :8], y[:, 8:], z(8, 3, 4, 3), z(1, 2, 3, 3), z(1, 2, 3), z(1, 2, 3, 3), z(1, 2, 3, 3),
                         z(1, 2, 3), z(1, 3, 3), 1, 2, (1.0,) * 3, (0.0,) * 3, (2,) * 3, (2, 2, 2))
    (name, args), = [c for c in fake.calls if c[0] == "occ_lift_splat_fused"]
    assert args[:4] == (y.data_ptr(), 24 * 12, y[:, 8:].data_ptr(), 24 * 12)
