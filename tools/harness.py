"""What the bench tools share: the card line they print and the loop that times the ways of doing one job against each other.
Scripts in this directory import it as a sibling (`from harness import card, timed`)."""
import subprocess
import time

import numpy as np


def card(*fields):
    """The first GPU's name and power limit, then any further --query-gpu `fields`, as nvidia-smi prints them; "unknown" without it."""
    q = subprocess.run(["nvidia-smi", "--query-gpu=" + ",".join(("name", "power.limit") + fields), "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def timed(ways, warmup, rounds, checks=None):
    """ways: name -> call.  Each way is called `warmup` times, way after way; then every round calls the ways in order, each call
    timed alone with the host clock.  checks: name -> check of that way's output, run after each of its timed calls, outside the
    timed region.  Returns ms per way ({"median", "min", "max"} over the rounds) and, per checked way, whether every check held."""
    checks = checks or {}
    for fn in ways.values():
        for _ in range(warmup):
            fn()
    ms = {k: [] for k in ways}
    ok = {k: True for k in checks}
    for _ in range(rounds):
        for name, fn in ways.items():
            t0 = time.perf_counter()
            fn()
            ms[name].append(1e3 * (time.perf_counter() - t0))
            if name in checks:
                ok[name] &= bool(checks[name]())
    return {k: {"median": float(np.median(v)), "min": float(min(v)), "max": float(max(v))} for k, v in ms.items()}, ok
