"""Extracts the geo filter known answers of the reference into tests/golden/geo_filter_goldens.json (re-run: byte-identical):

* crates/milli/src/test_index.rs test_basic_geo_bounding_box: its documents (string and number coordinates), the eight
  `_geoBoundingBox` candidate sets and the two top-below-bottom errors;
* crates/milli/src/search/facet/filter/tests.rs: zero_radius (documents and ids), the `_geoRadius` / `_geoBoundingBox` cases of
  not_filterable (with and without other filterable attributes), the latitude / longitude errors of geo_radius_error and
  geo_bounding_box_error;
* crates/milli/tests/search/filters.rs geo_radius / not_geo_radius: keyword searches of TEST_QUERY over tests/assets/test_set.ndjson
  (criteria Words, Typo, Proximity, Attribute, Exactness; the synonyms of setup_search_index_with_criteria; TermsMatchingStrategy
  Last; limit 17), the asserted id set (expected_order of every document filtered by execute_filter's geo_rank thresholds) and each
  document's `_geo`, title and description;
* crates/meilisearch/tests/search/geo.rs: geo_bounding_box_with_string_and_number (GEO_DOCUMENTS of tests/common/mod.rs, hit ids,
  estimatedTotalHits) and geo_sort_with_geo_strings (status 200).

Error messages keep their first line only (the second is the filter's span).  External ids map to docids in insertion order.

usage: python tests/golden/extract_geo_filter_goldens.py <meilisearch checkout>"""
import json
import os
import re
import sys


def rust_docs(body):
    d = re.search(r"documents!\(\[(.*?)\]\)\)", body, re.S).group(1).replace("RESERVED_GEO_FIELD_NAME", '"_geo"')
    return json.loads("[" + re.sub(r",(\s*[}\]])", r"\1", d.rstrip().rstrip(",")) + "]")


def fn_body(src, name):
    start = src.index(f"fn {name}()")
    nxt = src.find("#[test]", start)
    return src[start: nxt if nxt >= 0 else len(src)]


def bounding_box(src):
    body = fn_body(src, "test_basic_geo_bounding_box")
    cases, errors = [], []
    for m in re.finditer(r'Filter::from_str\("([^"]+)"\).*?(?:@"RoaringBitmap<\[([\d, ]*)\]>"|@r###"\s*(.*?)\n)', body, re.S):
        if m.group(2) is not None:
            cases.append({"filter": m.group(1), "ids": [int(x) for x in m.group(2).split(",") if x.strip()]})
        else:
            errors.append({"filter": m.group(1), "message": m.group(3).strip()})
    return {"name": "test_basic_geo_bounding_box", "docs": rust_docs(body), "cases": cases, "errors": errors}


def filter_errors(src, name):
    body = fn_body(src, name)
    return [{"filter": f, "message": msg.strip()}
            for f, msg in re.findall(r'Filter::from_str\("(_geo[^"]+)"\).*?snapshot!\(error\.to_string\(\), @r"\s*(.*?)\n', body, re.S)]


def not_filterable(src):
    body = fn_body(src, "not_filterable")
    split = body.index("set_filterable_fields")
    out = []
    for f, msg, at in ((m.group(1), m.group(2), m.start()) for m in
                       re.finditer(r'Filter::from_str\("(_geo[^"]+)"\).*?snapshot!\(error\.to_string\(\), @r"\s*(.*?)\n', body, re.S)):
        out.append({"filter": f, "message": msg.strip(), "other_filterable": ["title"] if at > split else []})
    return out


def zero_radius(src):
    body = fn_body(src, "zero_radius")
    f = re.search(r'Filter::from_str\("([^"]+)"\)', body).group(1)
    ids = [int(x) for x in re.search(r"assert_eq!\(documents_ids, vec!\[([\d, ]*)\]\)", body).group(1).split(",")]
    docs = [{"id": d["id"], "_geo": d["_geo"]} for d in rust_docs(body)]
    return {"name": "zero_radius", "docs": docs, "filter": f, "ids": ids}


def keyword(ref):
    base = os.path.join(ref, "crates/milli/tests")
    filters = open(os.path.join(base, "search/filters.rs")).read()
    mod = open(os.path.join(base, "search/mod.rs")).read()
    content = open(os.path.join(base, "assets/test_set.ndjson")).read()
    dec, docs, i = json.JSONDecoder(), [], 0
    while True:
        while i < len(content) and content[i].isspace():
            i += 1
        if i >= len(content):
            break
        d, i = dec.raw_decode(content, i)
        docs.append(d)
    query = re.search(r'pub const TEST_QUERY: &str = "([^"]+)";', mod).group(1)
    synonyms = {a: [b] for a, b in re.findall(r'S\("(\w+)"\) => vec!\[S\("([\w ]+)"\)\]', mod)}
    cases = []
    for name in ("geo_radius", "not_geo_radius"):
        f = re.search(r"test_filter!\(\s*" + name + r',\s*vec!\[Right\("([^"]+)"\)\]', filters).group(1)
        prefix = "NOT _geoRadius" if f.startswith("NOT") else "_geoRadius"
        op, bound = re.search(r'filter\.starts_with\("' + prefix + r'"\) \{\s*id = \(document\.geo_rank ([<>]) (\d+)\)', mod).groups()
        ids = sorted(d["id"] for d in docs if (d["geo_rank"] < int(bound) if op == "<" else d["geo_rank"] > int(bound)))
        cases.append({"name": name, "filter": f, "ids": ids})
    return {"query": query, "criteria": ["words", "typo", "proximity", "attribute", "exactness"], "terms_matching_strategy": "last",
            "limit": 17, "searchable": ["title", "description"], "synonyms": synonyms,
            "docs": [{"id": d["id"], "title": d["title"], "description": d["description"], "_geo": d["_geo"]} for d in docs],
            "cases": cases}


def meilisearch(ref):
    common = open(os.path.join(ref, "crates/meilisearch/tests/common/mod.rs")).read()
    geo_rs = open(os.path.join(ref, "crates/meilisearch/tests/search/geo.rs")).read()
    block = re.search(r"pub static GEO_DOCUMENTS: Lazy<Value> = Lazy::new\(\|\| \{\s*json!\((\[.*?\])\)\s*\}\);", common, re.S).group(1)
    docs = [{"id": d["id"], **({"_geo": d["_geo"]} if "_geo" in d else {})} for d in json.loads(block)]
    box = geo_rs[geo_rs.index("async fn geo_bounding_box_with_string_and_number"):]
    box = box[: box.index("#[actix_rt::test]")]
    sort = geo_rs[geo_rs.index("async fn geo_sort_with_geo_strings"):]
    sort = sort[: sort.index("#[actix_rt::test]")]
    return {"docs": docs,
            "geo_bounding_box_with_string_and_number": {
                "filter": re.search(r'"filter": "([^"]+)"', box).group(1),
                "ids": [int(x) for x in re.findall(r'^\s{22}"id": (\d+),', box, re.M)],
                "estimated_total_hits": int(re.search(r'"estimatedTotalHits": (\d+)', box).group(1))},
            "geo_sort_with_geo_strings": {
                "filter": re.search(r'"filter": "([^"]+)"', sort).group(1),
                "sort": json.loads(re.search(r'"sort": (\[.*?\])', sort).group(1)),
                "status": int(re.search(r"assert_eq!\(code, (\d+)", sort).group(1))}}


def main(ref):
    test_index = open(os.path.join(ref, "crates/milli/src/test_index.rs")).read()
    tests_rs = open(os.path.join(ref, "crates/milli/src/search/facet/filter/tests.rs")).read()
    out = {"source": "crates/milli/src/test_index.rs, crates/milli/src/search/facet/filter/tests.rs, crates/milli/tests/search/"
                     "filters.rs, crates/meilisearch/tests/search/geo.rs (v1.50.0)",
           "bounding_box": bounding_box(test_index),
           "zero_radius": zero_radius(tests_rs),
           "not_filterable": not_filterable(tests_rs),
           "range_errors": filter_errors(tests_rs, "geo_radius_error") + filter_errors(tests_rs, "geo_bounding_box_error"),
           "keyword": keyword(ref),
           "meilisearch": meilisearch(ref)}
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "geo_filter_goldens.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True, ensure_ascii=False)
        f.write("\n")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "/root/reference")
