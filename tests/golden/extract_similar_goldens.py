"""Extracts the `/similar` known answers of the reference into tests/golden/similar_goldens.json (re-run: byte-identical):

* crates/meilisearch/tests/similar/mod.rs: the five DOCUMENTS (external id, release_year, the 3-d `manual` vector) in insertion order,
  so internal docid = position;
* the requests of the tests `basic`, `ranking_score_threshold`, `filter` and `limit_and_offset`, each with the external ids of its
  snapshot's hits in order, their `_rankingScore` when the snapshot shows it, and `estimatedTotalHits` when the snapshot has it.

usage: python tests/golden/extract_similar_goldens.py <meilisearch checkout>"""
import json
import os
import re
import sys

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "similar_goldens.json")
TESTS = ("basic", "ranking_score_threshold", "filter", "limit_and_offset")


def strip_comments(s):
    return re.sub(r"//[^\n]*", "", s)


def documents(src):
    block = re.search(r"static DOCUMENTS: Lazy<Value> = Lazy::new\(\|\| \{\s*json!\((\[.*?\])\)\s*\}\);", src, re.S).group(1)
    block = re.sub(r",(\s*[}\]])", r"\1", strip_comments(block))  # trailing commas are legal in json! but not in JSON
    return [{"id": d["id"], "release_year": d["release_year"], "vector": d["_vectors"]["manual"]} for d in json.loads(block)]


def test_bodies(src):
    """name -> body of each `async fn name()`"""
    heads = list(re.finditer(r"async fn (\w+)\(\)", src))
    return {m.group(1): src[m.end():(heads[i + 1].start() if i + 1 < len(heads) else len(src))] for i, m in enumerate(heads)}


def cases(name, body):
    out = []
    calls = list(re.finditer(r"\.similar\(\s*json!\((\{.*?\})\),", body, re.S))
    for i, m in enumerate(calls):
        rest = body[m.end():(calls[i + 1].start() if i + 1 < len(calls) else len(body))]
        req = json.loads(m.group(1))
        hits = re.search(r'json_string!\(response\["hits"\]\), @(?:r###"(.*?)"###|"(.*?)")\);', rest, re.S)
        hits = json.loads(hits.group(1) if hits.group(1) is not None else hits.group(2))
        total = re.search(r'json_string!\(response\["estimatedTotalHits"\]\), @"(\d+)"\);', rest)
        out.append({"test": name, "request": req, "hits": [h["id"] for h in hits],
                    "scores": [h["_rankingScore"] for h in hits] if hits and all("_rankingScore" in h for h in hits) else None,
                    "estimatedTotalHits": int(total.group(1)) if total else None})
    return out


def main(root):
    src = open(os.path.join(root, "crates", "meilisearch", "tests", "similar", "mod.rs")).read()
    bodies = test_bodies(src)
    out = {"documents": documents(src), "cases": [c for t in TESTS for c in cases(t, bodies[t])]}
    with open(OUT, "w") as f:
        f.write(json.dumps(out, ensure_ascii=False, sort_keys=True, separators=(",", ":")) + "\n")


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    main(sys.argv[1])
