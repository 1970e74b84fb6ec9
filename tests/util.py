import os

import numpy as np
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

# north_star tolerance: 1e-3 relative fp32 per output tensor (SURVEY.md 8(d))
RTOL = 1e-3


def golden(name):
    return np.load(os.path.join(GOLDEN, name))


def parity_log(line):
    """Print a parity line; with OCC_PARITY_LOG=<file> also append it there (the suite writes nothing by default)."""
    print(line)
    log = os.environ.get("OCC_PARITY_LOG")
    if log:
        os.makedirs(os.path.dirname(os.path.abspath(log)), exist_ok=True)
        with open(log, "a") as f:
            f.write(line + "\n")


def rel_err(a, b):
    """max|a-b| / max|b| (per-tensor relative error)."""
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def rel_rms(a, b):
    """||a-b||_2 / ||b||_2 (per-tensor relative RMS error)."""
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).pow(2).sum().sqrt() / b.pow(2).sum().sqrt().clamp_min(1e-30))


def allclose_violations(a, b, tol=RTOL):
    """SURVEY.md 8(d), second criterion: allclose(rtol=tol, atol=tol * rms(b)); returns the number of violating elements."""
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    rms = float(b.pow(2).mean().sqrt())
    return int(((a - b).abs() > tol * rms + tol * b.abs()).sum())


def assert_close(a, b, tol=RTOL, what=""):
    """The tolerance of every floating-point parity test, exactly as SURVEY.md 8(d) fixes it -- per output tensor BOTH
        max|a-b| / max|b| <= tol                         (north_star: 1e-3 relative fp32)   and
        allclose(a, b, rtol=tol, atol=tol * rms(b))      (no element off by more than tol*(rms + |b|)).
    OCC_PARITY_REPORT_ONLY=1 logs the numbers without asserting (used to record a before/after table)."""
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    assert a.shape == b.shape, f"{what}: shape {tuple(a.shape)} vs {tuple(b.shape)}"
    assert torch.isfinite(a).all(), f"{what}: non-finite values"
    r, q, nv = rel_err(a, b), rel_rms(a, b), allclose_violations(a, b, tol)
    line = f"[parity] {what}: rel_max {r:.2e} rel_rms {q:.2e} allclose_violations {nv}/{a.numel()} (tol {tol:.0e})"
    parity_log(line)
    if os.environ.get("OCC_PARITY_REPORT_ONLY") != "1":
        assert r <= tol and nv == 0, f"{what}: rel_max {r:.3e}, rel_rms {q:.3e}, allclose violations {nv} (tol {tol:.0e})"
    return r


def round_tf32(t):
    i = t.clone().contiguous().view(torch.int32)
    i.add_(0x1000).bitwise_and_(-8192)
    return i.view(torch.float32)


class FakeLibrary:
    """Stand-in for libocc_b200.so (monkeypatch it over ops.lib): every function the header declares records its
    arguments and returns 0, so a call that gets past the argument checks of ops is recorded instead of launched."""

    def __init__(self):
        from occformer_b200 import _lib
        self.calls = []
        for name in _lib.signatures():
            setattr(self, name, lambda *args, name=name: self.calls.append((name, args)) or 0)
