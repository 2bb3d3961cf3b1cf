"""Extracts the facet search known answers of the reference into tests/golden/facet_search_goldens.json (re-run: byte-identical).

From crates/meilisearch/tests/search/facet_search.rs: every test that indexes the shared `DOCUMENTS` (or its own `documents`
literal) with `genres` filterable and asserts on a facet search over all documents: the documents' `genres`, the settings that
change the answer (`maxValuesPerFacet`, `sortFacetValuesBy`, typo tolerance `enabled`, `disableOnWords`), each `facetQuery`, and
what is asserted: the number of hits, the leading hits, or the `facetHits` snapshot.

Not extracted, and why:
* test_settings_documents_indexing_swapping_and_facet_search and the tests built on it: they index `NESTED_DOCUMENTS` and check
  settings swaps, distinct or locales, which the library does not take part in;
* non_filterable_facet_search_error and the `facetSearch` on/off tests: the facet-searchable check and the `facetSearch` setting
  stay with the caller;
* facet_search_with_filterable_attributes_rules: its cases turn on the rule matching (patterns, `facetSearch: false` per rule),
  which stays with the caller as well;
* distinct_facet_search_on_movies: distinct inside facet search is not built.

usage: python tests/golden/extract_facet_search_goldens.py <meilisearch checkout>"""
import json
import os
import re
import sys


def rust_json(lit):
    """a `json!` literal with Rust's trailing commas -> Python"""
    return json.loads(re.sub(r",(\s*[}\]])", r"\1", lit))


def bracketed(src, at):
    """the text of the [...] starting at src[at] == '['"""
    depth = 0
    for i in range(at, len(src)):
        depth += {"[": 1, "]": -1}.get(src[i], 0)
        if depth == 0:
            return src[at:i + 1]
    raise ValueError("unbalanced")


def tests(src):
    """(name, body) of every #[actix_rt::test]"""
    starts = [m.start() for m in re.finditer(r"#\[actix_rt::test\]\s*async fn (\w+)", src)]
    for a, b in zip(starts, starts[1:] + [len(src)]):
        body = src[a:b]
        yield re.search(r"async fn (\w+)", body).group(1), body


def main(root):
    path = os.path.join(root, "crates", "meilisearch", "tests", "search", "facet_search.rs")
    src = open(path).read()
    shared = rust_json(bracketed(src, src.index("json!([", src.index("static DOCUMENTS")) + 6))
    out = {"source": "crates/meilisearch/tests/search/facet_search.rs", "cases": []}
    for name, body in tests(src):
        if "facet_search(json!" not in body or "update_settings_filterable_attributes" not in body:
            continue
        if "facetSearch" in body or "update_settings(json!" in body:
            continue  # the caller's facetSearch setting and rule matching
        if "distinct" in body.lower():
            continue  # distinct inside facet search is not built
        own = re.search(r"let documents = json!\(\[", body)
        docs = rust_json(bracketed(body, own.end() - 1)) if own else shared
        if "DOCUMENTS.clone()" not in body and not own:
            continue
        settings = {"max_values": 100, "order": "alpha", "typos": True, "exact_words": []}
        m = re.search(r'"maxValuesPerFacet": (\d+)', body)
        if m:
            settings["max_values"] = int(m.group(1))
        if re.search(r'"sortFacetValuesBy": \{ "\*": "count" \}', body):
            settings["order"] = "count"
        if re.search(r'typo_tolerance\(json!\(\{ "enabled": false \}\)\)', body):
            settings["typos"] = False
        m = re.search(r'"disableOnWords": (\[[^\]]*\])', body)
        if m:
            settings["exact_words"] = json.loads(m.group(1))
        calls = list(re.finditer(r"facet_search\(json!\((\{.*?\})\)\)", body, re.S))
        for i, c in enumerate(calls):
            req = json.loads(c.group(1))
            rest = body[c.end(): calls[i + 1].start() if i + 1 < len(calls) else len(body)]
            case = dict(test=name, facet=req["facetName"], query=req.get("facetQuery"), **settings)
            case["genres"] = [d.get(req["facetName"], []) for d in docs]
            m = re.search(r'(?:as_array\(\)\.unwrap\(\)\.len\(\), @"(\d+)"|as_array\(\)\.unwrap\(\)\.len\(\), (\d+)\)|hits\.len\(\), (\d+)\))', rest)
            if m:
                case["n_hits"] = int(next(g for g in m.groups() if g))
            lead = re.findall(r'assert_eq!\(hits\[(\d+)\], json!\((\{.*?\})\)\)', rest)
            if lead:
                case["leading_hits"] = [[json.loads(j)["value"], json.loads(j)["count"]] for _, j in lead]
            m = re.search(r'snapshot!\(response\["facetHits"\], @r###"(.*?)"###\)', rest, re.S)
            if m:
                case["hits"] = [[h["value"], h["count"]] for h in json.loads(m.group(1))]
            if len(case) > len(settings) + 4:
                out["cases"].append(case)
    dst = os.path.join(os.path.dirname(os.path.abspath(__file__)), "facet_search_goldens.json")
    with open(dst, "w") as f:
        json.dump(out, f, indent=1, ensure_ascii=False, sort_keys=True)
        f.write("\n")
    print(f"{len(out['cases'])} cases -> {dst}")


if __name__ == "__main__":
    main(sys.argv[1])
