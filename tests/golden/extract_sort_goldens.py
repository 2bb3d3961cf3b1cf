"""Extracts the Sort known answers of the reference into tests/golden/sort_goldens.json (re-run: byte-identical):
crates/milli/src/search/new/tests/sort.rs — the index of create_index(), the four searches of test_sort and the one of
test_redacted with their inline documents_ids snapshots, and the Sort score values of snapshots/*sort__sort-{2,5,8,11}.snap.

usage: python tests/golden/extract_sort_goldens.py <meilisearch checkout>"""
import json
import os
import re
import sys


def main(ref):
    base = os.path.join(ref, "crates/milli/src/search/new/tests")
    src = open(os.path.join(base, "sort.rs")).read()
    docs = re.search(r"documents!\(\[(.*?)\]\)\)", src, re.S).group(1)
    docs = json.loads("[" + re.sub(r",(\s*[}\]])", r"\1", docs.rstrip().rstrip(",")) + "]")
    cases = []
    test_sort = src[src.index("fn test_sort()"): src.index("fn test_redacted()")]
    for i, m in enumerate(re.finditer(r"sort_criteria\(vec!\[(.*?)\]\);.*?documents_ids:\?\}\"\), @\"(\[.*?\])\"", test_sort, re.S)):
        sort = [f"{f}:{d.lower()}" for d, f in re.findall(r"AscDesc::(Asc|Desc)\(Member::Field\(S\(\"(\w+)\"\)\)\)", m.group(1))]
        snap = open(os.path.join(base, "snapshots", f"milli__search__new__tests__sort__sort-{3 * i + 2}.snap")).read()
        values = []
        for v in re.findall(r"value: (Null|String\(\"[^\"]*\"\)|Number\([^)]*\))", snap):
            values.append(None if v == "Null" else (v[8:-2] if v.startswith("String") else float(v[7:-1])))
        cases.append({"name": f"test_sort_{i}", "sort": sort, "ids": json.loads(m.group(2)), "sort_values": values})
    red = src[src.index("fn test_redacted()"):]
    m = re.search(r"sort_criteria\(vec!\[(.*?)\]\);.*?documents_ids:\?\}\"\), @\"(\[.*?\])\"", red, re.S)
    sort = [f"{f}:{d.lower()}" for d, f in re.findall(r"AscDesc::(Asc|Desc)\(Member::Field\(S\(\"(\w+)\"\)\)\)", m.group(1))]
    cases.append({"name": "test_redacted", "sort": sort, "ids": json.loads(m.group(2)), "sort_values": None})
    out = {"source": "crates/milli/src/search/new/tests/sort.rs (v1.50.0)", "criteria": ["sort"], "limit": 20, "docs": docs, "cases": cases}
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "sort_goldens.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "/root/reference")
