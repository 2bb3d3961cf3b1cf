"""CPU: the facet specification (tests/facet_spec.py) against the reference's own answers (tests/golden/facet_goldens.json, written
by tests/golden/extract_facet_goldens.py), and the library's f64 Display formatter against the specification's port."""
import hashlib
import os
import shutil
import subprocess

import pytest

from tests.facet_fixtures import case_candidates, golden_facets, load_facet_goldens
from tests.facet_spec import debug_string, facet_stats, facet_values, rust_f64_display, stats_debug_string

G = load_facet_goldens()
MILLI = [(t["name"], i) for t in G["milli"] for i, c in enumerate(t["cases"]) if c["order"] == "alpha"]


@pytest.mark.parametrize("name,i", MILLI)
def test_facet_distribution_rs(name, i):
    t = next(x for x in G["milli"] if x["name"] == name)
    c = t["cases"][i]
    fac = golden_facets(t)
    fid = fac.fields[t["field"]]
    cand = case_candidates(c)
    if c["call"] == "compute_stats":
        got = "{}" if cand is None else stats_debug_string(t["field"], facet_stats(fac, fid, cand))
    else:
        got = debug_string(t["field"], facet_values(fac, fid, cand, c["max_values"], documents=range(len(t["docs"]))))
    assert (hashlib.md5(got.encode()).hexdigest() if c["md5"] else got) == c["expect"]


def test_server_cases():
    mv, casing = G["server"]
    fac = golden_facets(mv)
    for c in mv["cases"]:
        got = facet_values(fac, fac.fields["number"], set(range(len(mv["docs"]))), c["max_values"])
        assert len(got) == c["len"]
    fac = golden_facets(casing)
    assert dict(facet_values(fac, fac.fields["dog"], {0})) == casing["facet_distribution"]["dog"]


VALUES = [0.0, -0.0, 1.5, 0.1, 1e16, 1e21, 1e23, 2.0 ** 60, 1.2345678901234567e25, 1.7976931348623157e308, 5e-324, -3.25e-7, 123456.789]


@pytest.mark.skipif(shutil.which("g++") is None, reason="needs a host C++ compiler")
def test_library_display_formatter(tmp_path):
    """rust_f64_display of host_index.cpp (which orders the <= 3000 path's numbers) prints what the specification's port prints"""
    csrc = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "meilisearch_b200", "csrc")
    main = tmp_path / "main.cpp"
    main.write_text('#include <cstdio>\n#include <cstdlib>\n#include "host_index.h"\n'
                    "int main(int c, char **v) { for (int i = 1; i < c; i++) printf(\"%s\\n\", b200::rust_f64_display(strtod(v[i], nullptr)).c_str()); }\n")
    exe = tmp_path / "display"
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I", csrc, str(main), os.path.join(csrc, "host_index.cpp"), "-o", str(exe), "-pthread"])
    out = subprocess.run([str(exe)] + [repr(v) for v in VALUES], capture_output=True, text=True, check=True).stdout.split("\n")[:-1]
    assert out == [rust_f64_display(v) for v in VALUES]
