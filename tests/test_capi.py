"""C-ABI library: loads, exports every symbol include/quatro_b200.h declares, and fails loudly without a GPU
(no CPU fallback).  No compute calls here -- those are the -m gpu parity tests."""
import ctypes as C
import re
from pathlib import Path

import pytest

from quatro_b200 import capi

ROOT = Path(__file__).resolve().parent.parent


def declared_symbols():
    txt = (ROOT / "include" / "quatro_b200.h").read_text()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(qb200_[a-z_0-9]+)\s*\(", txt)))


def test_header_symbols_are_exported():
    lib = capi.load_library()
    names = declared_symbols()
    assert len(names) >= 20
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/quatro_b200.h but not exported"
    assert sorted(capi.EXPORTED_SYMBOLS) == names, "capi.py binding list and header disagree"
    assert lib.qb200_version() == 100


def test_default_params_match_python_mirror():
    lib = capi.load_library()
    p = capi.Params()
    lib.qb200_default_params(C.byref(p))
    q = capi.default_params()
    assert bytes(p) == bytes(q)
    # config/params.yaml values
    assert (round(p.voxel_size, 6), round(p.normal_radius, 6), round(p.fpfh_radius, 6)) == (0.3, 0.5, 0.75)
    assert (p.noise_bound, p.cbar2, p.rotation_max_iterations, p.rotation_gnc_factor, p.rotation_cost_threshold) == (0.3, 1.0, 50, 1.4, 0.00011)
    assert p.inlier_selection_mode == capi.PMC_HEU and p.cote_mode == capi.COTE_MEDIAN
    c = capi.Config()
    lib.qb200_default_config(C.byref(c))
    assert bytes(c) == bytes(capi.default_config())


def test_struct_layouts():
    assert C.sizeof(capi.Result) == 56 + 8 + 128 + 0 or C.sizeof(capi.Result) == capi.RESULT_DTYPE.itemsize
    assert C.sizeof(capi.Pair) == 24
    assert C.sizeof(capi.Params) % 8 == 0


def test_no_cpu_fallback_without_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present: the failure path is exercised on the CPU-only box")
    with pytest.raises(capi.QuatroB200Error) as e:
        capi.Handle()
    assert e.value.code == -2  # QB200_ERR_NO_DEVICE


def test_product_does_not_reference_the_oracle():
    """The product path must never import, link or call the test oracle."""
    for f in list((ROOT / "quatro_b200").rglob("*.py")) + list((ROOT / "quatro_b200" / "csrc").glob("*")) + list((ROOT / "include").rglob("*.h*")):
        txt = f.read_text(errors="ignore")
        assert "quatro_oracle" not in txt and "from oracle" not in txt and "import oracle" not in txt and "qo_" not in txt.replace("qo_math", ""), f


POD_MIRRORS = {"qb200_params": capi.Params, "qb200_config": capi.Config, "qb200_result": capi.Result, "qb200_pair": capi.Pair,
               "qb200_patchwork_params": capi.PatchworkParams, "qb200_segment_params": capi.SegmentParams,
               "qb200_preprocess_out": capi.PreprocessOut, "qb200_corr_set": capi.CorrSet, "qb200_pair_lists": capi.PairLists}


def header_fields(struct):
    """Member names of `typedef struct <struct> { ... } <struct>;` in include/quatro_b200.h, in declaration order."""
    hdr = (ROOT / "include" / "quatro_b200.h").read_text()
    body = hdr[hdr.index(f"typedef struct {struct} {{"):hdr.index(f"}} {struct};")].split("{", 1)[1]
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    return [n for decl in body.split(";") for n in re.findall(r"(\w+)\s*(?:\[\w*\])?\s*(?:,|$)", decl.strip())]


@pytest.fixture(scope="module")
def pod_probe(tmp_path_factory):
    """sizeof and every member's offsetof of each mirrored POD, and QB200_FLAG_LISTS_TRUNCATED, from a C compiler."""
    import subprocess
    tmp = tmp_path_factory.mktemp("pod")
    lines = [f'  printf("{t} %zu\\n", sizeof({t}));\n' +
             "".join(f'  printf("{t}.{f} %zu\\n", offsetof({t}, {f}));\n' for f, _ in m._fields_) for t, m in POD_MIRRORS.items()]
    (tmp / "pod.c").write_text('#include <stddef.h>\n#include <stdio.h>\n#include "quatro_b200.h"\nint main(void) {\n' + "".join(lines) +
                               '  printf("QB200_FLAG_LISTS_TRUNCATED %d\\n", (int)QB200_FLAG_LISTS_TRUNCATED);\n  return 0;\n}\n')
    r = subprocess.run(["/usr/bin/gcc", "-std=c11", "-Wall", "-Werror", f"-I{ROOT / 'include'}", str(tmp / "pod.c"), "-o", str(tmp / "pod")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return {k: int(v) for k, v in (ln.split() for ln in subprocess.run([str(tmp / "pod")], capture_output=True, text=True,
                                                                         check=True).stdout.splitlines())}


@pytest.mark.parametrize("struct", list(POD_MIRRORS))
def test_pod_layouts_match_the_header(pod_probe, struct):
    """The ctypes mirror of a POD of include/quatro_b200.h has the header's members, in order, at the offsets a C compiler gives
    them, and the same size."""
    mirror = POD_MIRRORS[struct]
    fields = [f for f, _ in mirror._fields_]
    assert fields == header_fields(struct)
    assert C.sizeof(mirror) == pod_probe[struct]
    for f in fields:
        assert getattr(mirror, f).offset == pod_probe[f"{struct}.{f}"], f
    if struct == "qb200_pair_lists":
        assert pod_probe["QB200_FLAG_LISTS_TRUNCATED"] == capi.FLAG_LISTS_TRUNCATED
        assert set(capi.LIST_LAYOUT) == set(fields) - {"cap_per_pair", "kind"}
