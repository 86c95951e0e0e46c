#!/usr/bin/env python3
"""Two scans through qb200_patchwork + qb200_segment_cloud (a small workload for profiling the pre-processing kernels); prints one
JSON line shaped like a bench line that labels the run."""
import json
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from quatro_b200 import synth  # noqa: E402
from quatro_b200.capi import Handle, default_patchwork_params, default_segment_params  # noqa: E402

pp, sp = default_patchwork_params(), default_segment_params()
with Handle(max_batch_slots=2) as h:
    for seed in (1, 2):
        src = synth.outdoor_pair(seed)[0]
        g, ng, st = h.patchwork(src, pp)
        v, o = h.segment_cloud(ng, sp)
print(json.dumps({"config": {"workload": f"one 64-ring scan ({len(src)} points) through qb200_patchwork + qb200_segment_cloud"},
                  "points": len(src), "ground": len(g), "nonground": len(ng), "valid": len(v), "outliers": len(o)}))
