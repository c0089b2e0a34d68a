"""What the benchmark scripts under tools/ share: the repository and tests/ (where the oracles' scene builders live) on
sys.path, the card a run is timed on, CUDA-event timing, kernel-launch counts and the JSON rows.  The scripts run as
`python tools/<name>.py`, so tools/ is on the path and `import benchkit` finds this module; import it before the
project's own modules.
"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (os.path.join(ROOT, "tests"), ROOT):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from demon_b200 import _lib   # noqa: E402


def device_info():
    """Name, power limit and maximum SM clock of the card torch times on (its current device), to be read in the same run
    as the timings.  nvidia-smi numbers cards on its own and ignores CUDA_VISIBLE_DEVICES, so the card is selected by
    its UUID.  A query that fails gives "unknown (<exception class>)": the timings are still measurements."""
    props = torch.cuda.get_device_properties(torch.cuda.current_device())
    info = {"gpu": props.name}
    try:
        out = subprocess.run(["nvidia-smi", "-i", "GPU-%s" % props.uuid, "--query-gpu=power.limit,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30, check=True).stdout
        info["power_limit"], info["max_sm_clock"] = (s.strip() for s in out.strip().splitlines()[0].split(","))
    except Exception as e:
        info["power_limit"] = info["max_sm_clock"] = "unknown (%s)" % type(e).__name__
    return info


def _event():
    return torch.cuda.Event(enable_timing=True)


def call_times(fn, reps, warmup=3, sync_each=True):
    """Milliseconds of each of `reps` calls of fn after `warmup` untimed ones, each call bracketed by CUDA events on the
    current stream.  sync_each waits for every call before issuing the next; otherwise all calls are queued and waited
    for once."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    events = [(_event(), _event()) for _ in range(reps)]
    for a, b in events:
        a.record()
        fn()
        b.record()
        if sync_each:
            b.synchronize()
    torch.cuda.synchronize()
    return [a.elapsed_time(b) for a, b in events]


def span_ms(fn, reps, warmup=3):
    """Mean milliseconds per call of `reps` back-to-back calls of fn after `warmup` untimed ones: one CUDA-event span
    around them all."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = _event(), _event()
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def summary(times):
    """Median, min and max of per-call milliseconds, and how many calls they are."""
    return dict(ms=float(np.median(times)), ms_min=float(np.min(times)), ms_max=float(np.max(times)), steps=len(times))


def device_events(fn):
    """fn's result and the device activity of one call of it (kernels, memsets and copies of every library), recorded by
    torch.profiler after the device is idle."""
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    return out, [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


def profiled_kernels(fn):
    """Kernels one call of fn launches, torch's and every library's, counted by torch.profiler (copies and memsets not)."""
    return sum(1 for e in device_events(fn)[1] if not e.name.startswith(("Memcpy", "Memset")))


def library_launches(fn):
    """Kernels this library launches in one call of fn, by its own counter (demon_launch_count); torch's ops in fn are
    not counted."""
    lib = _lib.load()
    n0 = lib.demon_launch_count()
    fn()
    return int(lib.demon_launch_count() - n0)


class Rows(list):
    """A run's JSON rows.  add() merges device_info() into a row, prints it and keeps it; save() appends the rows to
    `out`, if given, once the run is through, so a run that fails part way writes nothing."""

    def __init__(self, out):
        super().__init__()
        self.out, self.info = out, device_info()

    def add(self, row):
        row.update(self.info)
        print(json.dumps(row), flush=True)
        self.append(row)

    def save(self):
        if self.out:
            os.makedirs(os.path.dirname(os.path.abspath(self.out)), exist_ok=True)
            with open(self.out, "a") as f:
                f.writelines(json.dumps(r) + "\n" for r in self)
