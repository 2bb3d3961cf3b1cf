"""CPU specification of the facet distribution and facet stats: a literal port of FacetDistribution::facet_values (both paths) and
compute_stats (crates/milli/src/search/facet/facet_distribution.rs:110-337, facet_distribution_iter.rs:26-232, facet/mod.rs:39-59)
over a FacetImage's dicts.  It never goes through the library."""
import decimal

CANDIDATES_THRESHOLD = 3000


def rust_f64_display(x):
    """`impl Display for f64`: shortest round-trip digits, never an exponent"""
    if x != x:
        return "NaN"
    if x in (float("inf"), float("-inf")):
        return "inf" if x > 0 else "-inf"
    s = format(decimal.Decimal(repr(float(x))), "f")
    return s.rstrip("0").rstrip(".") if "." in s else s


def _hits(docs, cand):
    return sorted(d for d in set(docs) if d in cand)


def facet_values(facets, fid, candidates, max_values=100, documents=None):
    """facet_values(field_id, OrderBy::Lexicographic) over `candidates` (a set of docids) -> list of (key, count).  candidates None:
    none were given, so the facet levels are walked over `documents` (documents_ids) whatever its size"""
    cand = set(documents if candidates is None else candidates)
    nums = facets.numbers.get(fid, {})
    strs = facets.strings.get(fid, {})
    dist = {}  # IndexMap<String, u64>: insertion order, an insert on an existing key overwrites its value in place
    if candidates is not None and len(cand) <= CANDIDATES_THRESHOLD:
        # facet_distribution_from_documents, Number: a BTreeMap keyed by value.to_string(), extended with the first max - len
        lex = {}
        for v, docs in nums.items():
            c = len(_hits(docs, cand))
            if c:
                lex[rust_f64_display(v)] = lex.get(rust_f64_display(v), 0) + c
        for k in sorted(lex)[: max(0, max_values - len(dist))]:
            dist[k] = lex[k]
        # String: a BTreeMap keyed by the normalised value holding the original of the first candidate (in docid order) that has it
        norm = {}
        for v, docs in strs.items():
            h = _hits(docs, cand)
            if h:
                norm[v] = (facets.originals.get((fid, h[0], v), v), len(h))
        for v in sorted(norm, key=lambda x: x.encode())[: max(0, max_values - len(dist))]:
            orig, c = norm[v]
            dist[orig] = c
    else:
        # facet levels: numbers in numeric order, then strings in byte order; insert, then break when the map holds max_values
        for v in sorted(nums):
            c = len(_hits(nums[v], cand))
            if not c:
                continue
            dist[rust_f64_display(v)] = c
            if len(dist) == max_values:
                break
        for v in sorted(strs, key=lambda x: x.encode()):
            h = _hits(strs[v], cand)
            if not h:
                continue
            dist[facets.originals.get((fid, h[0], v), v)] = len(h)
            if len(dist) == max_values:
                break
    return list(dist.items())


def facet_stats(facets, fid, candidates):
    """compute_stats for one field: (facet_min_value, facet_max_value) over the candidates, None without a number value"""
    cand = set(candidates)
    vals = [v for v, docs in facets.numbers.get(fid, {}).items() if any(d in cand for d in docs)]
    return (min(vals), max(vals)) if vals else None


def debug_string(field, pairs):
    """`{:?}` of the BTreeMap<String, IndexMap<String, u64>> FacetDistribution::execute returns for one field"""
    return "{" + f'"{field}": {{' + ", ".join(f'"{k}": {c}' for k, c in pairs) + "}}"


def stats_debug_string(field, stats):
    """`{:?}` of compute_stats' BTreeMap<String, (f64, f64)> for one field"""
    return "{}" if stats is None else "{" + f'"{field}": ({stats[0]!r}, {stats[1]!r})' + "}"
