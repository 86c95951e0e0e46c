"""Every CUDA resource of a handle and its lanes (device and pinned memory, streams, events) is held by an owner type of
csrc/owners.cuh, which releases it in its destructor.  Outside that header no source allocates or releases one by hand,
so there is no hand-kept release list that a new buffer could be missing from."""
import re
from pathlib import Path

CSRC = Path(__file__).resolve().parent.parent / "quatro_b200" / "csrc"
OWNERS = "owners.cuh"
RAW_CALLS = re.compile(r"\b(cudaFree|cudaFreeHost|cudaStreamDestroy|cudaEventDestroy|cudaMalloc|cudaMallocHost)\s*\(")


def _sources():
    files = sorted(p for p in CSRC.iterdir() if p.suffix in (".cu", ".cuh"))
    assert any(p.name == OWNERS for p in files), files
    return [p for p in files if p.name != OWNERS]


def test_no_raw_allocation_or_release_outside_the_owners():
    found = []
    for p in _sources():
        for n, line in enumerate(p.read_text().splitlines(), 1):
            for m in RAW_CALLS.finditer(line):
                found.append(f"{p.name}:{n}: {m.group(1)}")
    assert not found, "\n".join(found)


def test_no_hand_written_release_lists():
    for p in _sources():
        text = p.read_text()
        for name in ("lane_free", "cache_free"):
            assert not re.search(rf"\b{name}\b", text), f"{p.name} still has {name}"
