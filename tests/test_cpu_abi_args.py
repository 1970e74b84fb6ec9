"""Tensor arguments of the C ABI are checked against their pointer declarations in include/occ_b200.h before anything is
enqueued.  The library is replaced by a recording fake: a check that regresses shows up as a recorded call, never as a
kernel reading a host pointer."""
import pytest
import torch

from util import FakeLibrary


@pytest.fixture
def fake(monkeypatch):
    from occformer_b200 import ops
    f = FakeLibrary()
    monkeypatch.setattr(ops, "lib", lambda: f)
    return f


def test_header_parser_pointee_types(tmp_path):
    from occformer_b200 import _lib
    params = _lib.parameters()
    assert params["occ_mask_bits"] == [("pooled", "int"), ("bits", "unsigned"), ("B", None), ("S", None), ("Q", None),
                                       ("stream", None)]
    assert params["occ_ssc_counts"] == [("pred", "unsigned char"), ("target", "unsigned char"), ("n", None),
                                        ("K", None), ("ignore", None), ("conf_ws", "long long"), ("out", "long long"),
                                        ("stream", None)]
    conv = dict(params["occ_conv_bf16x3"])
    assert (conv["x"], conv["gn_stats"], conv["workspace"], conv["workspace_bytes"]) == ("float", "double", "void", None)
    assert params["occ_voxel_pool_workspace_layout"] == [("n_points", None), ("B", None), ("X", None), ("Y", None),
                                                         ("Z", None), ("off_counts", "size_t"), ("off_head", "size_t"),
                                                         ("off_next", "size_t"), ("off_vox_id", "size_t")]
    assert params["occ_version"] == []
    bad = tmp_path / "bad.h"
    bad.write_text("int occ_ok(const float* x, int n);\nint occ_bad(const short* x, int n);\n")
    with pytest.raises(RuntimeError, match="occ_bad"):
        _lib.parameters(str(bad))


def _cpu_args(params, at):
    """arguments of a declaration without its stream: a CPU tensor of the declared pointee type at index `at`, NULL at
    the other pointers, 0 for the values"""
    from occformer_b200 import ops
    args = [None if pointee else 0 for _, pointee in params[:-1]]
    args[at] = torch.zeros(4, dtype=ops._DTYPES[params[at][1]] or torch.uint8)
    return args


def test_every_pointer_rejects_a_cpu_tensor(fake):
    from occformer_b200 import _lib, ops
    checked = 0
    for name, params in _lib.parameters().items():
        if not params or params[-1][0] != "stream":
            continue
        for i, (param, pointee) in enumerate(params):
            if pointee is None:
                continue
            with pytest.raises(RuntimeError, match=rf"{name}\({param}\) must be a CUDA tensor \(no CPU fallback"):
                ops._call(name, *_cpu_args(params, i))
            checked += 1
    assert checked > 200 and fake.calls == []


def test_tensor_at_a_value_or_host_parameter_is_rejected(fake):
    from occformer_b200 import ops
    t = torch.zeros(4, dtype=torch.int32)
    with pytest.raises(RuntimeError, match=r"occ_mask_bits\(S\) is not a device pointer"):
        ops._call("occ_mask_bits", None, None, 1, t, 1)
    with pytest.raises(RuntimeError, match=r"occ_voxel_pool_workspace_layout\(off_head\) is not a device pointer"):
        ops._call("occ_voxel_pool_workspace_layout", 1, 1, 1, 1, 1, None, torch.zeros(1, dtype=torch.int64), None, None)
    assert fake.calls == []


def test_previously_unchecked_wrappers_reject_cpu_tensors(fake):
    from occformer_b200 import ops
    z = torch.zeros
    B, grid, Q, E, NC = 1, (2, 2, 2), 4, 32, 3
    W = {k: z(E, E) for k in ("pn_w", "pn_b", "clsT", "cls_b", "m0T", "m0b", "m1T", "m1b", "m2T", "m2b")}
    L = {k: z(E, E) for k in ("ca_woT", "ca_bo", "n0w", "n0b", "sa_inT", "sa_inb", "sa_woT", "sa_bo", "n1w", "n1b",
                              "f1T", "f2T", "f2b")}
    L["f1b"] = z(2 * E)
    calls = {
        "occ_classmix": lambda: ops.classmix(z(B, 8, Q), z(B, Q, NC), B, grid, grid, Q, NC, with_labels=True),
        "occ_query_head": lambda: ops.query_head(z(B * Q, E), W, NC),
        "occ_cross_merge": lambda: ops.cross_merge(z(B, 1, 1, Q, 34), 1, 1, z(B * Q, E), z(Q, E), Q, L, 1.0),
        "occ_self_attn_ffn": lambda: ops.self_attn_ffn(z(B * Q, 3 * E), z(B * Q, E), Q, L, 1),
        "occ_mask_pool": lambda: ops.mask_pool(z(B, 8, Q), B, grid, (1, 1, 1), Q),
        "occ_mask_gemm_pool": lambda: ops.mask_gemm_pool(z(B, 8, E), z(B * Q, E), B, grid, (1, 1, 1), Q),
        "occ_gn_relu_zmean_ln": lambda: ops.gn_relu_zmean_ln(z(B * 8, E), z(B, 1, 2, dtype=torch.float64), z(E), z(E),
                                                             z(E), z(E), B, 4, 2, E, 1),
        "occ_dualpath_fuse": lambda: ops.dualpath_fuse(z(B * 8, E), z(B * 4, E), z(E), 0.0, z(B * 8, E), B, 4, 2, E),
        "occ_lift_splat_fused": lambda: ops.lift_splat_fused(
            z(1, 16, 2, 2)[:, :8], z(1, 16, 2, 2)[:, 8:], z(8, 2, 2, 3), z(1, 1, 3, 3), z(1, 1, 3), z(1, 1, 3, 3),
            z(1, 1, 3, 3), z(1, 1, 3), z(1, 3, 3), 1, 1, (1.0,) * 3, (0.0,) * 3, (2,) * 3, (2, 2, 2)),
    }
    for name, call in calls.items():
        with pytest.raises(RuntimeError, match=rf"{name}\(\w+\) must be a CUDA tensor \(no CPU fallback"):
            call()
    assert fake.calls == []
