"""How the benchmark scripts measure: the card line, CUDA-graph capture, torch arms with TF32 allowed or disabled, the
alternated L2-flushed replay loop, the relative error and the GPU time per kind of launch.  A module, not a script."""
import collections
import subprocess

import torch


def card():
    """name, power limit and max SM clock of the GPU, read from nvidia-smi in the same run as the numbers they qualify"""
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown card"


def graphed(fn):
    """-> (a CUDA graph of fn, its output) after two warm-up calls on a side stream"""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = fn()
    torch.cuda.synchronize()
    return g, out


def torch_arms(fn):
    """fn, a torch forward, as the arms torch_tf32 (torch's default torch.backends.cudnn.allow_tf32 = True) and
    torch_fp32 (TF32 disabled for cuDNN and matmul), each under no_grad.  They set the flags when called; capture()
    restores them."""
    matmul = torch.backends.cuda.matmul.allow_tf32

    def arm(allow):
        def run():
            torch.backends.cudnn.allow_tf32 = allow
            torch.backends.cuda.matmul.allow_tf32 = allow and matmul
            with torch.no_grad():
                return fn()
        return run
    return {"torch_tf32": arm(True), "torch_fp32": arm(False)}


def capture(arms):
    """{name: fn} -> ({name: CUDA graph}, {name: output}), with the TF32 flags as they were before"""
    tf32 = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    graphs, outs = {}, {}
    for name, fn in arms.items():
        graphs[name], outs[name] = graphed(fn)
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32
    return graphs, outs


def alternated(graphs, iters, warmup):
    """warmup + iters rounds, each replaying every graph in turn after zeroing 128 MiB (more than the 50 MiB L2), timed
    by a pair of CUDA events per replay -> {name: [ms per replay of the last iters rounds]}"""
    flush = torch.empty(128 * 1024 * 1024 // 4, dtype=torch.float32, device="cuda")
    times = {k: [] for k in graphs}
    for it in range(warmup + iters):
        for name, gr in graphs.items():
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            gr.replay()
            e1.record()
            e1.synchronize()
            if it >= warmup:
                times[name].append(e0.elapsed_time(e1))
    return times


def rel(a, b):
    """max|a-b| / max|b|"""
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def launch_shares(fn, kinds):
    """The library's launch count over one eager call of fn (torch.profiler) and its GPU time per kind of launch, in ms:
    kinds is ((kind, "name|name"), ...), the first kind with a name in the kernel's name wins, else "other"."""
    from torch.profiler import ProfilerActivity, profile
    from occformer_b200 import ops
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        n0 = ops.LAUNCH_COUNT[0]
        fn()
        torch.cuda.synchronize()
        launches = ops.LAUNCH_COUNT[0] - n0
    t = collections.defaultdict(float)
    cnt = collections.Counter()
    for e in prof.events():
        if not str(e.device_type).endswith("CUDA"):
            continue
        kind = next((k for k, pat in kinds if any(p in e.name for p in pat.split("|"))), "other")
        t[kind] += e.device_time_total / 1e3 if hasattr(e, "device_time_total") else e.cuda_time_total / 1e3
        cnt[kind] += 1
    total = sum(t.values())
    return launches, {k: {"launches": cnt[k], "ms": round(t[k], 3), "share": round(t[k] / total, 4)} for k in t}
