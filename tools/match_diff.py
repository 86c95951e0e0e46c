"""Triage: compare the tensor-core matcher with the oracle on the batch-test pairs, dump the first differing pair."""
import sys
import tempfile
from pathlib import Path
sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import numpy as np
from quatro_b200 import capi, synth
from oracle.oracle_lib import Oracle

def main():
    o = Oracle(); o.set_num_threads(16)
    p = capi.default_params(); p.use_tuple_test = 0
    h = capi.Handle(max_batch_slots=2)
    out = {}
    for rep in range(1):
        for seed in range(10, 21):
            src, tgt = synth.outdoor_pair(seed, rings=32, azimuths=900)[:2]
            sv = o.voxelize(src, p.voxel_size, 1)[0]; tv = o.voxelize(tgt, p.voxel_size, 1)[0]
            fa = o.compute_fpfh(sv, p.normal_radius, p.fpfh_radius, p.fpfh_radius)[1]
            fb = o.compute_fpfh(tv, p.normal_radius, p.fpfh_radius, p.fpfh_radius)[1]
            ref = o.match(sv, fa, tv, fb, p)
            got = h.match(sv, fa, tv, fb, p)
            same = np.array_equal(got[0], ref[0]) and got[1] == ref[1]
            print("rep", rep, "seed", seed, "n_mutual", got[1], ref[1], "same" if same else "DIFF", flush=True)
            if not same and "fa" not in out:
                out = dict(fa=fa, fb=fb, got=got[0], ref=ref[0], seed=seed)
    if out:
        dst = Path(tempfile.gettempdir()) / "match_diff.npz"
        np.savez(dst, **out)
        print("first differing pair written to", dst)
    print("stats", h.debug_match_stats())

if __name__ == "__main__":
    main()
