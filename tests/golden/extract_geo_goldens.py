"""Extracts the GeoSort known answers of the reference into tests/golden/geo_sort_goldens.json (re-run: byte-identical):
crates/milli/src/search/new/tests/geo_sort.rs — per placeholder test its documents (external ids map to docids in insertion order),
every search's sort list and inline ids snapshot, and the GeoSort values (each hit's bucket point, or None) of the matching
snapshots/*geo_sort*.snap; the invariants of test_geo_sort_reached_max_bucket_size; the three `_geoDistance` values of
crates/meilisearch/tests/search/geo.rs geo_sort_with_words.  geo_sort_mixed_with_words searches with query terms: out of scope.

usage: python tests/golden/extract_geo_goldens.py <meilisearch checkout>"""
import json
import os
import re
import sys

SNAP = "milli__search__new__tests__geo_sort__{}-{}.snap"


def docs_of(body):
    d = re.search(r"documents!\(\[(.*?)\]\)\)", body, re.S).group(1).replace("RESERVED_GEO_FIELD_NAME", '"_geo"')
    return json.loads("[" + re.sub(r",(\s*[}\]])", r"\1", d.rstrip().rstrip(",")) + "]")


def sort_list(src):
    out = []
    for d, kind, arg in re.findall(r"AscDesc::(Asc|Desc)\(Member::(Geo|Field)\((.*?)\)\)", src):
        if kind == "Geo":
            lat, lng = [float(x) for x in arg.strip("[]").split(",")]
            out.append(f"_geoPoint({lat}, {lng}):{d.lower()}")
        else:
            out.append(f"{re.search(chr(34) + r'(\w+)' + chr(34), arg).group(1)}:{d.lower()}")
    return out


def snap_values(base, test, k):
    snap = open(os.path.join(base, "snapshots", SNAP.format(test[len("test_"):], k))).read()
    vals = []
    for m in re.finditer(r"value: (None|Some\(\s*\[\s*([-\d.e]+),\s*([-\d.e]+),?\s*\]\s*,?\s*\))", snap):
        vals.append(None if m.group(1) == "None" else [float(m.group(2)), float(m.group(3))])
    return vals


def main(ref):
    base = os.path.join(ref, "crates/milli/src/search/new/tests")
    src = open(os.path.join(base, "geo_sort.rs")).read()
    fns = {m.group(1): m.start() for m in re.finditer(r"fn (\w+)\(\)", src)}
    names = sorted(fns, key=fns.get)
    body = {n: src[fns[n]: (fns[names[i + 1]] if i + 1 < len(names) else len(src))] for i, n in enumerate(names)}
    tests = []
    for test in ("test_geo_sort", "test_geo_sort_with_following_ranking_rules", "test_geo_sort_around_the_edge_of_the_flat_earth"):
        b = body[test]
        docs = docs_of(b)
        cases, k = [], 0
        for m in re.finditer(r"sort_criteria\(vec!\[(.*?)\]\);.*?\{ids:\?\}\"\), @\"(\[.*?\])\"\);\s*insta::assert_snapshot!\(format!\(\"\{scores:#\?\}\"\)\);",
                             b, re.S):
            k += 2
            ext = json.loads(m.group(2))
            docid = {d["id"]: i for i, d in enumerate(docs)}
            cases.append({"sort": sort_list(m.group(1)), "ids": [docid[x] for x in ext], "geo_values": snap_values(base, test, k)})
        tests.append({"name": test, "docs": docs, "cases": cases})
    mb = body["test_geo_sort_reached_max_bucket_size"]
    maxb = {"name": "test_geo_sort_reached_max_bucket_size", "docs": docs_of(mb), "max_bucket_size": 2, "sort": sort_list(mb),
            "strategies": [["iterative", 1000], ["rtree", 1000]], "first_6_ids_in": [6, 11], "next_4_ids_in": [12, 15],
            "no_geo_ids": [int(x) for x in re.findall(r'"(\d+)"', re.search(r"no_geo_ids:\?\}\"\), @r#\"(\[.*?\])\"#", mb).group(1))]}
    geo_rs = open(os.path.join(ref, "crates/meilisearch/tests/search/geo.rs")).read()
    w = geo_rs[geo_rs.index("async fn geo_sort_with_words()"):]
    w = w[: w.index("async fn", 10)] if "async fn" in w[10:] else w
    dist = [int(x) for x in re.findall(r'"_geoDistance": (\d+)', w)]
    pts = [[float(a), float(b)] for a, b in re.findall(r'"lat": (-?\d+), "lng": (-?\d+) \}', w)]
    ids = [int(x) for x in re.findall(r'"id": (\d+),\n\s*"doggo"', w)]
    out = {"source": "crates/milli/src/search/new/tests/geo_sort.rs, crates/meilisearch/tests/search/geo.rs (v1.50.0)",
           "criteria": ["words", "sort"], "tests": tests, "max_bucket": maxb,
           "geo_distance": {"target": [0.0, 0.0], "points": [pts[i] for i in ids], "rounded_metres": dist},
           "out_of_scope": {"geo_sort_mixed_with_words": "keyword search (query terms) with a GeoSort rule"}}
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "geo_sort_goldens.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "/root/reference")
