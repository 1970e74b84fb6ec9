import copy
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from occformer_b200 import ops  # loads no library: ops.lib() does that on its first call

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden")

# north_star tolerance: 1e-3 relative fp32 per output tensor (SURVEY.md 8(d))
RTOL = 1e-3
SENTINEL = 0x7FC0FFEE  # a NaN: an output row left unwritten also fails the finiteness check of assert_close


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


def bits(t):
    return t.detach().contiguous().view(torch.int32).cpu()


# ------------------------------------------------------------------ one C-ABI entry point at a time
def _int_view(t):
    """t's bits as integers of its element width, on its device (the outputs compared are up to hundreds of MB)"""
    return t.contiguous().view({4: torch.int32, 8: torch.int64}[t.element_size()])


def sentinel(rows, cols, device):
    """a (rows, cols) fp32 tensor of SENTINEL bits"""
    return torch.full((rows, cols), SENTINEL, dtype=torch.int32, device=device).view(torch.float32)


def untouched(t, what):
    assert bool((_int_view(t) == SENTINEL).all()), f"{what}: written outside the output"


def same_bits(a, b, what):
    assert torch.equal(_int_view(a), _int_view(b)), f"{what}: not bit-identical"


def launches(name, *args):
    """ops._call(name, *args) -> the number of kernels and memsets the entry point enqueued"""
    n0 = ops.LAUNCH_COUNT[0]
    ops._call(name, *args)
    return ops.LAUNCH_COUNT[0] - n0


def rejected(name, *args, buffers=(), rc=None):
    """ops._call(name, *args) fails -- rc None: it raises; rc -2: it returns -2 under unsupported_ok (an unsupported
    shape); any other rc: it raises as argument error rc -- enqueues nothing and leaves every buffer as it was"""
    before = [_int_view(b).clone() for b in buffers]
    n0 = ops.LAUNCH_COUNT[0]
    if rc == -2:
        assert ops._call(name, *args, unsupported_ok=True) == rc
    else:
        with pytest.raises(RuntimeError, match=None if rc is None else f"argument error {rc}"):
            ops._call(name, *args)
    torch.cuda.synchronize()
    assert ops.LAUNCH_COUNT[0] == n0, f"{name}: enqueued work before rejecting the call"
    for b, b0 in zip(buffers, before):
        assert torch.equal(_int_view(b), b0), f"{name}: a rejected call changed a buffer"


def misaligned(t):
    """a flat view of t's storage from 4 bytes in (for a freshly allocated t: 4 bytes past a 16-byte boundary), for calls
    that must reject it before touching it (t itself can then be checked for being unchanged)"""
    return t.reshape(-1)[1:]


def graph_replay(fn, outs):
    """fn() captured into a CUDA graph on a side stream, the tensors of outs filled with SENTINEL, the graph replayed ->
    outs after the replay.  outs is read after the capture, so fn may append the outputs it allocates."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s), torch.cuda.graph(graph, stream=s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    for t in outs:
        t.view(torch.int32).fill_(SENTINEL)
    graph.replay()
    torch.cuda.synchronize()
    return outs


def images(n, H, W, seed=0):
    return torch.randn(n, 3, H, W, generator=torch.Generator().manual_seed(seed))


def f64(net, device=None):
    """The same module in float64 in eval mode (the oracle of the GPU tests), on the host, or on `device` when given.
    .cpu() drops the prepared-parameter cache, so the copy carries no CUDA state."""
    ref = copy.deepcopy(net).cpu().double().eval()
    return ref if device is None else ref.to(device)


def trace(fn):
    """One call of fn under torch.profiler -> dict(counted: the library's launch count over the call (ops.LAUNCH_COUNT),
    kernels / memsets: the occ:: kernels and memsets of the trace, other: the names of any other GPU work)"""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        n0 = ops.LAUNCH_COUNT[0]
        fn()
        torch.cuda.synchronize()
        counted = ops.LAUNCH_COUNT[0] - n0
    gpu = [e.name for e in prof.events() if str(e.device_type).endswith("CUDA")]
    return dict(counted=counted, kernels=sum("occ::" in e for e in gpu), memsets=sum(e.startswith("Memset") for e in gpu),
                other=sorted({e for e in gpu if "occ::" not in e and not e.startswith("Memset")}))


def run_script(script, *args, timeout):
    """python tests/<script> <args> in a process of its own, with this interpreter's flags: its profiler session and
    graph capture must not change what a later profiler session of this process records (test_gpu_launch_count compares
    a trace with the launch counter).  -> the JSON of its last output line"""
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable, *flags, os.path.join(HERE, script), *args], capture_output=True, text=True,
                       timeout=timeout)
    assert r.returncode == 0, f"{' '.join([script, *args])} failed:\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}"
    return json.loads(r.stdout.strip().splitlines()[-1])


def run_trace(case, timeout):
    """tests/forward_trace.py <case> by run_script.  Asserts that the forward ran only library kernels and memsets.
    -> its result"""
    res = run_script("forward_trace.py", case, timeout=timeout)
    print(f"[{case} launches] counted {res['counted']}, trace: {res['kernels']} occ:: kernels + {res['memsets']} memsets")
    assert not res["other"], f"non-library GPU work: {res['other'][:5]}"
    return res


class FakeLibrary:
    """Stand-in for libocc_b200.so (monkeypatch it over ops.lib): every function the header declares records its
    arguments and returns 0, so a call that gets past the argument checks of ops is recorded instead of launched."""

    def __init__(self):
        from occformer_b200 import _lib
        self.calls = []
        for name in _lib.signatures():
            setattr(self, name, lambda *args, name=name: self.calls.append((name, args)) or 0)
