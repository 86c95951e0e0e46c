"""The single-pair stage calls (csrc/stages.cu) move the wave counters through the lane's pinned mirror of the counter block: one
read_counters copy per call brings every count back, and write_counter sets a count without a wait of its own.  No source keeps
a helper that copies one counter and waits for it, and stages.cu copies no counter by hand."""
import re
from pathlib import Path

CSRC = Path(__file__).resolve().parent.parent / "quatro_b200" / "csrc"
STAGES = CSRC / "stages.cu"
DELETED = ("get_counter", "set_counter", "copy_ints", "fetch_result", "match_result", "download_corr", "upload_matched",
           "upload_cloud_as_voxels")
# a cudaMemcpy* call whose arguments name a field of the device counters (L->ctr.n_vox, ...), over line breaks too
COUNTER_COPY = re.compile(r"cudaMemcpy\w*\([^;]*\bctr\.")


def test_single_counter_helpers_are_gone():
    found = []
    for p in sorted(CSRC.iterdir()):
        if p.suffix in (".cu", ".cuh"):
            text = p.read_text()
            found += [f"{p.name}: {name}" for name in DELETED if re.search(rf"\b{name}\b", text)]
    assert not found, "\n".join(found)


def test_stage_calls_copy_counters_only_through_the_mirror():
    text = STAGES.read_text()
    assert "read_counters" in text and "write_counter" in text
    found = [text[m.start():text.index(";", m.start()) + 1] for m in COUNTER_COPY.finditer(text)]
    assert not found, "\n".join(found)
