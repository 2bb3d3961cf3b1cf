"""Extracts the filter known answers of the reference into tests/golden/filter_goldens.json (re-run: byte-identical):

* crates/milli/tests/search/filters.rs: every `test_filter!` case (name and the `Vec<Either<Vec<&str>, &str>>` it builds: an AND of
  its entries, each a filter string or an OR of filter strings), and the id set tests/search/mod.rs expected_filtered_ids computes for
  it over crates/milli/tests/assets/test_set.ndjson, with execute_filter ported line by line below;
* the documents of test_set.ndjson in file order (docid = position) and the filterable attributes of
  setup_search_index_with_criteria.

usage: python tests/golden/extract_filter_goldens.py <meilisearch checkout>"""
import json
import os
import re
import sys
import unicodedata

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "filter_goldens.json")


def normalize_facet(s):
    return unicodedata.normalize("NFKD", s.strip()).lower()


def rust_u32(s):
    return int(s) if re.fullmatch(r"\+?\d+", s) and int(s) < 2 ** 32 else None


def is_empty_value(v):
    return isinstance(v, (str, list, dict)) and len(v) == 0


def contains_key_rec(v, key):
    if isinstance(v, list):
        return any(contains_key_rec(x, key) for x in v)
    if isinstance(v, dict):
        return any(k == key or contains_key_rec(x, key) for k, x in v.items())
    return False


def contains_null_rec(v, key):
    if isinstance(v, dict):
        return any((k == key and x is None) or contains_null_rec(x, key) for k, x in v.items())
    if isinstance(v, list):
        return any(contains_null_rec(x, key) for x in v)
    return False


MISSING = object()


def execute_filter(f, d):
    """tests/search/mod.rs execute_filter: the document's id when it passes, else None"""
    opt1, opt12, ok = d.get("opt1", MISSING), d.get("opt1.opt2", MISSING), False
    if "!=" in f:
        field, v = f.split("!=", 1)
        ok = (field == "tag" and d["tag"] != v) or (field == "asc_desc_rank" and d["asc_desc_rank"] != rust_u32(v))
    elif "=" in f:
        field, v = f.split("=", 1)
        ok = (field == "tag" and d["tag"] == v) or (field == "asc_desc_rank" and d["asc_desc_rank"] == int(v))
    elif "STARTS WITH" in f:
        field, prefix = f.split("STARTS WITH", 1)
        value = {"tag": d["tag"], "title": d["title"], "description": d["description"]}[field.strip()]
        ok = normalize_facet(value).startswith(normalize_facet(prefix.strip().strip("'")))
    elif "<" in f and f.split("<", 1)[0] == "asc_desc_rank":
        ok = d["asc_desc_rank"] < int(f.split("<", 1)[1])
    elif ">" in f and f.split(">", 1)[0] == "asc_desc_rank":
        ok = d["asc_desc_rank"] > int(f.split(">", 1)[1])
    elif f.startswith("_geoRadius"):
        ok = d["geo_rank"] < 100000
    elif f.startswith("NOT _geoRadius"):
        ok = d["geo_rank"] > 1000000
    elif f in ("opt1 EXISTS", "NOT opt1 NOT EXISTS"):
        ok = opt1 is not MISSING
    elif f in ("NOT opt1 EXISTS", "opt1 NOT EXISTS"):
        ok = opt1 is MISSING
    elif f == "opt1.opt2 EXISTS":
        ok = opt12 is not MISSING or (opt1 is not MISSING and contains_key_rec(opt1, "opt2"))
    elif f in ("opt1 IS NULL", "NOT opt1 IS NOT NULL"):
        ok = opt1 is not MISSING and opt1 is None
    elif f in ("NOT opt1 IS NULL", "opt1 IS NOT NULL"):
        ok = opt1 is MISSING or opt1 is not None
    elif f == "opt1.opt2 IS NULL":
        ok = (opt12 is not MISSING and opt12 is None) or (opt1 is not MISSING and opt1 is not None and contains_null_rec(opt1, "opt2"))
    elif f in ("opt1 IS EMPTY", "NOT opt1 IS NOT EMPTY"):
        ok = opt1 is not MISSING and is_empty_value(opt1)
    elif f in ("NOT opt1 IS EMPTY", "opt1 IS NOT EMPTY"):
        ok = opt1 is MISSING or not is_empty_value(opt1)
    elif f == "opt1.opt2 IS EMPTY":
        ok = opt12 is not MISSING and is_empty_value(opt12)
    elif f in ("tag_in IN[1, 2, 3, four, five]", "NOT tag_in NOT IN[1, 2, 3, four, five]"):
        ok = d["id"] in ("A", "B", "C", "D", "E")
    elif f == "tag_in NOT IN[1, 2, 3, four, five]":
        ok = d["id"] not in ("A", "B", "C", "D", "E")
    else:
        raise ValueError(f"unknown filter {f!r}")
    return d["id"] if ok else None


def expected_filtered_ids(filters, docs):
    ids = {d["id"] for d in docs}
    for e in filters:
        if isinstance(e, list):
            sel = set().union(*({x for x in (execute_filter(f, d) for d in docs) if x} for f in e))
        else:
            sel = {x for x in (execute_filter(e, d) for d in docs) if x}
        ids &= sel
    return sorted(ids)


def main(ref):
    tests = os.path.join(ref, "crates", "milli", "tests")
    text = open(os.path.join(tests, "assets", "test_set.ndjson")).read()
    docs, at, dec = [], 0, json.JSONDecoder()
    while True:
        while at < len(text) and text[at].isspace():
            at += 1
        if at >= len(text):
            break
        d, at = dec.raw_decode(text, at)
        docs.append(d)
    src = open(os.path.join(tests, "search", "filters.rs")).read()
    cases = []
    for m in re.finditer(r"test_filter!\(\s*(\w+),\s*vec!\[(.*?)\]\s*\);", src, re.S):
        filters = []
        for it in re.finditer(r'Right\("((?:[^"\\]|\\.)*)"\)|Left\(vec!\[(.*?)\]\)', m.group(2), re.S):
            if it.group(1) is not None:
                filters.append(it.group(1))
            else:
                filters.append(re.findall(r'"((?:[^"\\]|\\.)*)"', it.group(2)))
        cases.append({"name": m.group(1), "filter": filters, "ids": expected_filtered_ids(filters, docs)})
    mod = open(os.path.join(tests, "search", "mod.rs")).read()
    filterable = re.findall(r'FilterableAttributesRule::Field\(S\("([^"]+)"\)\)', mod)
    out = {"source": "crates/milli/tests/search/filters.rs, tests/search/mod.rs, tests/assets/test_set.ndjson",
           "filterable": filterable, "docs": docs, "cases": cases}
    with open(OUT, "w") as f:
        f.write(json.dumps(out, ensure_ascii=False, sort_keys=True, separators=(",", ":")) + "\n")
    print(f"{len(cases)} cases, {len(docs)} documents -> {OUT}")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "/root/reference")
