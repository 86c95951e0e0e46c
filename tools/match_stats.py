"""Diagnostics: how often the tensor-core matcher needs the exact fp32 chain (run on the GPU box)."""
import sys
from pathlib import Path
sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import numpy as np
from quatro_b200 import capi, synth

def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 16
    pairs = [synth.outdoor_pair(1000 + i)[:2] for i in range(n)]
    h = capi.Handle(max_batch_slots=n)
    p = capi.default_params()
    h.debug_match_stats(True)
    res = h.register_batch(pairs, p)
    st = h.debug_match_stats(True)
    entries = float(np.sum(res["n_src_vox"].astype(np.float64) * res["n_tgt_vox"]))
    print("pairs", n, "entries %.3e" % entries, st)
    print("exact fraction %.4f%%  evals/tile %.1f" % (100.0 * st["exact_evals"] / entries, st["exact_evals"] / max(1, st["tiles"])))
    print("kernel ms", h.kernel_ms())

if __name__ == "__main__":
    main()
