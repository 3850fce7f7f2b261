"""What the benchmark tools share: the record of the card a run uses, the HBM peak they quote, and their CUDA timers.

Each timer keeps the methodology of the tools that use it; where tools differ (warm-up counts, repetitions, clock),
they say so through arguments."""
import statistics
import subprocess
import time

import torch

HBM_BYTES_PER_S = 3.35e12          # H100 SXM data-sheet HBM3 bandwidth for a card allowed up to 700 W; not measured


def card():
    """Name, power limit and max SM clock of torch device 0, the card the run uses.  nvidia-smi is asked by that card's
    UUID: its own indices follow PCI order, not CUDA_VISIBLE_DEVICES.  Without a working nvidia-smi the second field
    holds its error text or None."""
    q = ["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
         f"--id=GPU-{torch.cuda.get_device_properties(0).uuid}"]
    try:
        out = subprocess.run(q, capture_output=True, text=True, timeout=30)
        smi = out.stdout.strip() or out.stderr.strip() or None
    except (OSError, subprocess.SubprocessError) as exc:
        smi = f"unavailable: {exc!r}"
    return {"name": torch.cuda.get_device_name(0), "name_power_limit_max_sm_clock": smi}


def _events():
    return torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)


def event_ms(fn):
    """ms of one call of fn, between CUDA events, synchronised."""
    s, e = _events()
    s.record()
    fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e)


def per_call_ms(fn, reps, warmup):
    """ms of each of `reps` calls of fn, each between its own pair of events, after `warmup` calls and a synchronise.
    The calls are queued back to back: nothing waits for the device until the last one."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ev = [_events() for _ in range(reps)]
    for s, e in ev:
        s.record()
        fn()
        e.record()
    torch.cuda.synchronize()
    return [s.elapsed_time(e) for s, e in ev]


def launch_ms(calls, reps):
    """{name: median ms} of the launches in calls ({name: fn}): `reps` rounds, each timing every launch once by
    event_ms, in insertion order."""
    times = {k: [] for k in calls}
    for _ in range(reps):
        for k, fn in calls.items():
            times[k].append(event_ms(fn))
    return {k: statistics.median(v) for k, v in times.items()}


def mean_ms(fn, iters):
    """Mean ms per call of `iters` back-to-back calls of fn between one pair of events."""
    s, e = _events()
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def graph_us(fn, launches=20, replays=3):
    """us per launch of fn on the GPU alone, without Python, ctypes or descriptor-encode time: 3 eager warm-up calls,
    `launches` calls captured in one CUDA graph, one untimed replay, then events around `replays` replays.  Returns the
    time and the graph, which a caller may replay again."""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(launches):
            fn()
    graph.replay()
    torch.cuda.synchronize()
    return mean_ms(graph.replay, replays) / launches * 1e3, graph


def alternate(arms, steps, flush, clock):
    """{name: fn}: one warm-up call of each arm, then `steps` rounds in which each arm runs once, in turn, after `flush`
    bytes are written to push the previous arm's data out of L2 (outside the timed span).  clock "events" times each
    call between CUDA events; "host" on the host clock between two synchronises, so host work inside fn counts in full.
    Returns ({name: upper median ms}, {name: [ms per round]})."""
    assert clock in ("events", "host"), clock
    buf = torch.empty(flush, dtype=torch.uint8, device="cuda")
    for fn in arms.values():
        fn()
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for i in range(steps):
        for k, fn in arms.items():
            buf.fill_(i & 0xFF)
            if clock == "events":
                times[k].append(event_ms(fn))
                continue
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            times[k].append((time.perf_counter() - t0) * 1e3)
    return {k: sorted(v)[len(v) // 2] for k, v in times.items()}, times
