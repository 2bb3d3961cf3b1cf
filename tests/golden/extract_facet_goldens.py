"""Extracts the facet distribution known answers of the reference into tests/golden/facet_goldens.json (re-run: byte-identical):

* crates/milli/src/search/facet/facet_distribution.rs, the tests of `mod tests`: each test's documents (the `colour` values, from
  the `documents!` literal or from the loop that builds them) and every FacetDistribution call with its candidates (null: none
  given, i.e. documents_ids through the facet levels), maxValuesPerFacet, order, whether it is `execute` or `compute_stats`, and
  the snapshot: the `{:?}` string, or the md5 of it for the two 1000-value cases;
* crates/meilisearch/tests/search/mod.rs: faceting_max_values_per_facet (number = id * 10 over 10 000 documents, a placeholder
  search with maxValuesPerFacet 100 and then 10 000: the number of entries) and change_facet_casing (the document as it stands after
  its replacement, and the snapshot).

Not extracted: search_facet_distribution in crates/meilisearch/tests/search/mod.rs.  Its first case only asserts that `title`
has an entry in the shared test set, and its other cases facet nested objects (`doggos.name`, `doggos`), whose extraction is out
of scope here.

usage: python tests/golden/extract_facet_goldens.py <meilisearch checkout>"""
import json
import os
import re
import sys


def fn_body(src, name):
    start = src.index(f"fn {name}()")
    nxt = src.find("#[test]", start + 1)
    nxt2 = src.find("#[actix_rt::test]", start + 1)
    ends = [x for x in (nxt, nxt2) if x >= 0]
    return src[start: min(ends) if ends else len(src)]


def colour_docs(body):
    """the documents' `colour` values, from the literal or from the loop of the test"""
    m = re.search(r"documents!\(\[(.*?)\]\);", body, re.S)
    if m:
        docs = json.loads("[" + re.sub(r",(\s*[}\]])", r"\1", m.group(1).strip().rstrip(",")) + "]")
        return [d["colour"] for d in docs]
    n = int(re.search(r"for i in 0\.\.([\d_]+)", body).group(1).replace("_", ""))
    lit = re.search(r"let facet_values = \[(.*?)\];", body, re.S)
    if lit:
        values = json.loads("[" + lit.group(1) + "]")
    elif 'format!("{x:x}")' in body:
        k = int(re.search(r"\(0\.\.(\d+)\)\.map\(\|x\| format!", body).group(1))
        values = [format(x, "x") for x in range(k)]
    else:
        k = int(re.search(r"let facet_values = \(0\.\.(\d+)\)\.collect", body).group(1))
        values = list(range(k))
    mod = int(re.search(r"facet_values\[i % (\d+)\]", body).group(1))
    expr = re.sub(r"\s+", " ", re.search(r'"colour": (.*?),\n\s*\}\)', body, re.S).group(1)).strip()
    out = []
    for i in range(n):
        v = values[i % mod]
        if expr == f"facet_values[i % {mod}]":
            out.append(v)
        elif expr == f"[facet_values[i % {mod}], facet_values[i % {mod}] + 1000]":
            out.append([v, v + 1000])
        elif expr == f'[facet_values[i % {mod}], format!("{{}}", facet_values[i % {mod}] + 1000)]':
            out.append([v, str(v + 1000)])
        else:
            raise ValueError(f"unknown document expression {expr!r}")
    if "if i % 2 == 0" in body:  # facet_mixed_values: odd documents hold one string instead
        alt = int(re.search(r'format!\("\{\}", facet_values\[i % \d+\] \+ (\d+)\)', body.split("} else {")[1]).group(1))
        out = [out[i] if i % 2 == 0 else str(values[i % mod] + alt) for i in range(n)]
    return out


def cases(body):
    out = []
    for chunk in body.split("let map = FacetDistribution::new")[1:]:
        chunk = chunk.split("let map =")[0]
        order = re.search(r"OrderBy::(default\(\)|Count)", chunk).group(1)
        c = re.search(r"\.candidates\((.*?)\)\n", chunk)
        cand = None
        if c:
            r = re.fullmatch(r"\((\d[\d_]*)\.\.(\d[\d_]*)\)\.collect\(\)", c.group(1).strip())
            cand = {"range": [int(r.group(1).replace("_", "")), int(r.group(2).replace("_", ""))]} if r else \
                [int(x) for x in re.search(r"\[([\d, ]*)\]", c.group(1)).group(1).split(",")]
        mx = re.search(r"\.max_values_per_facet\((\d+)\)", chunk)
        snap = re.search(r'milli_snap!\(format!\("\{map:\?\}"\)(?:, "[^"]*")?, @(?:r###"(.*?)"###|"(.*?)")\);', chunk, re.S)
        expect = snap.group(1) if snap.group(1) is not None else snap.group(2)
        out.append({"order": "count" if order == "Count" else "alpha", "candidates": cand, "max_values": int(mx.group(1)) if mx else 100,
                    "call": "compute_stats" if ".compute_stats()" in chunk else "execute",
                    "md5": bool(re.fullmatch(r"[0-9a-f]{32}", expect)), "expect": expect})
    return out


def main(root):
    src = open(os.path.join(root, "crates/milli/src/search/facet/facet_distribution.rs")).read()
    tests = src[src.index("mod tests"):]
    milli = []
    for name in re.findall(r"#\[test\]\s*fn (\w+)\(\)", tests):
        body = fn_body(tests, name)
        milli.append({"name": name, "field": "colour", "docs": colour_docs(body), "cases": cases(body)})
    ms = open(os.path.join(root, "crates/meilisearch/tests/search/mod.rs")).read()
    body = fn_body(ms, "faceting_max_values_per_facet")
    n = int(re.search(r"\(0\.\.([\d_]+)\)\.map\(\|id\| json!\(\{ \"id\": id, \"number\": id \* (\d+) \}\)\)", body).group(1).replace("_", ""))
    mul = int(re.search(r'"number": id \* (\d+)', body).group(1))
    lens = [int(x.replace("_", "")) for x in re.findall(r"assert_eq!\(numbers\.len\(\), ([\d_]+)\)", body)]
    maxes = [100] + [int(x.replace("_", "")) for x in re.findall(r'"maxValuesPerFacet": ([\d_]+)', body)]
    server = [{"name": "faceting_max_values_per_facet", "field": "number", "docs": [i * mul for i in range(n)],
               "cases": [{"max_values": m, "len": ln} for m, ln in zip(maxes, lens)]}]
    body = fn_body(ms, "change_facet_casing")
    final = {}
    for arr in re.findall(r"add_documents\(\s*json!\((\[.*?\])\),", body, re.S):
        for d in json.loads(arr):
            final[d["id"]] = d
    snap = re.search(r'json_string!\(response\["facetDistribution"\]\), @r###"(.*?)"###', body, re.S).group(1)
    server.append({"name": "change_facet_casing", "field": "dog", "docs": [final[k]["dog"] for k in sorted(final)],
                   "facet_distribution": json.loads(snap)})
    out = {"source": "meilisearch v1.50.0 @ 5cb2f2e", "milli": milli, "server": server,
           "not_extracted": [{"name": "search_facet_distribution",
                              "reason": "asserts only that `title` has an entry, and facets nested objects (doggos.name, doggos)"}]}
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "facet_goldens.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=None, separators=(",", ":"))
        f.write("\n")


if __name__ == "__main__":
    main(sys.argv[1])
