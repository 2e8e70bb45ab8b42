"""Measuring helpers shared by the profile scripts.

Every number a profile script records comes through these: the card it was measured on, read in the same run; CUDA
events around back-to-back calls after a warm-up; CUDA-graph replay; a host clock bracketed by device synchronises;
variants alternated round by round so that drift on a shared machine spreads over all of them; medians. Each helper
takes its counts as arguments, so every script keeps its own.
"""
import json
import os
import statistics
import subprocess
import time

import torch


def card():
    """{"device": torch's name of the current GPU, "nvidia_smi": nvidia-smi's name, power limit and maximum SM clock of
    it}. A read-only query: it changes no setting. When nvidia-smi is missing or fails, "nvidia_smi" holds the error
    text, so a measurement never fails for want of it."""
    dev = torch.cuda.current_device()
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                            "-i", str(dev)], capture_output=True, text=True, timeout=30, check=True)
        smi = q.stdout.strip()
    except subprocess.CalledProcessError as e:
        smi = "nvidia-smi failed: %s %s" % (e, (e.stdout + e.stderr).strip())
    except (OSError, subprocess.SubprocessError) as e:
        smi = "nvidia-smi failed: %s" % e
    return {"device": torch.cuda.get_device_name(dev), "nvidia_smi": smi}


def event_ms(fn, calls, warmup):
    """ms per call of fn: CUDA events around `calls` back-to-back calls, after `warmup` calls and a synchronise.
    Without a warm-up there is no synchronise: the start event is stream-ordered, so work the caller queued just
    before (resetting the inputs of a per-call timing, say) stays outside the window and hides the host's launch of
    fn."""
    for _ in range(warmup):
        fn()
    if warmup:
        torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(calls):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / calls


def graphed(fn, warmup):
    """One call of fn captured into a CUDA graph, after `warmup` calls on a side stream (as torch.cuda.graph asks);
    returns the graph's replay."""
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(warmup):
            fn()
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    return g.replay


def graph_ms(fn, calls, replays, warmup):
    """Device ms per call of fn: `calls` calls captured into one CUDA graph after `warmup` eager calls, and CUDA events
    around `replays` replays of it after one warm replay. For kernels shorter than their launch from Python, where
    events around eager calls would time the host."""
    for _ in range(warmup):
        fn()

    def batch():
        for _ in range(calls):
            fn()
    return event_ms(graphed(batch, 0), replays, 1) / calls


def wall_ms(fn):
    """Host ms of one call of fn, between two device synchronises: for work that reads results back on the host."""
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return 1e3 * (time.perf_counter() - t0)


def alternate(fns, rounds, time_one, warmup=0):
    """{name: [time_one(fn) of each round]} for the variants {name: fn}, interleaved round by round, after `warmup`
    calls of each variant and a synchronise."""
    for fn in fns.values():
        for _ in range(warmup):
            fn()
    torch.cuda.synchronize()
    out = {k: [] for k in fns}
    for _ in range(rounds):
        for k, fn in fns.items():
            out[k].append(time_one(fn))
    return out


def summary(values):
    return {"median_ms": statistics.median(values), "min_ms": min(values)}


def emit(record, out=None):
    """Print the record as one JSON line; with `out`, also write it, indented, to that file."""
    if out:
        os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
        with open(out, "w") as f:
            json.dump(record, f, indent=1)
    print(json.dumps(record), flush=True)
