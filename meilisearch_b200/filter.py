"""A recursive-descent parser for the filter expressions the tests and benchmarks use (a subset of filter-parser's grammar), producing
the FilterCondition tree the library's filter programs encode (include/b200milli.h b200_filter_programs).

Trees are tuples: ("and", [children]), ("or", [children]), ("not", child), ("cond", field, op, [raw values]) with op one of
= != > >= < <= TO IN EXISTS NULL EMPTY CONTAINS STARTS_WITH, and ("geo", kind, [raw numbers]) with kind radius, radius_resolution,
bbox or polygon.  As filter-parser builds them: a chain of ANDs (ORs) is one node, `f NOT IN [..]`, `f NOT EXISTS`, `f IS NOT NULL`,
`f IS NOT EMPTY`, `f NOT CONTAINS v` and `f NOT STARTS WITH v` are NOT over the positive condition, `f != v` is its own leaf.
Anything outside this grammar raises ValueError."""
from __future__ import annotations

import re

_TOKEN = re.compile(r"""\s*(?:(?P<punct>>=|<=|!=|[()\[\],=<>])|'(?P<sq>(?:[^'\\]|\\.)*)'|"(?P<dq>(?:[^"\\]|\\.)*)"|(?P<word>[^\s()\[\],=!<>'"]+))""")
KEYWORDS = {"AND", "OR", "NOT", "TO", "IN", "EXISTS", "IS", "NULL", "EMPTY", "CONTAINS", "STARTS", "WITH"}
_GEO = {"_geoRadius": "radius", "_geoBoundingBox": "bbox", "_geoPolygon": "polygon"}


def _tokens(s):
    out, at = [], 0
    while at < len(s):
        if s[at:].strip() == "":
            break
        m = _TOKEN.match(s, at)
        if not m or m.end() == at:
            raise ValueError(f"filter: cannot read {s[at:]!r}")
        at = m.end()
        if m.group("punct"):
            out.append(("p", m.group("punct")))
        elif m.group("word") is not None:
            w = m.group("word")
            out.append(("k", w) if w in KEYWORDS else ("v", w))
        else:
            raw = m.group("sq") if m.group("sq") is not None else m.group("dq")
            out.append(("v", re.sub(r"\\(.)", r"\1", raw)))
    return out


class _Parser:
    def __init__(self, s):
        self.t, self.i = _tokens(s), 0

    def peek(self, k=0):
        return self.t[self.i + k] if self.i + k < len(self.t) else (None, None)

    def take(self, kind=None, text=None):
        tok = self.peek()
        if tok[0] is None or (kind and tok[0] != kind) or (text and tok[1] != text):
            raise ValueError(f"filter: expected {text or kind}, found {tok[1]!r}")
        self.i += 1
        return tok[1]

    def expr(self):
        return self.chain("OR", "or", self.conj)

    def conj(self):
        return self.chain("AND", "and", self.neg)

    def chain(self, word, name, sub):
        items = [sub()]
        while self.peek() == ("k", word):
            self.i += 1
            items.append(sub())
        return items[0] if len(items) == 1 else (name, items)

    def neg(self):
        if self.peek() == ("k", "NOT"):
            self.i += 1
            return ("not", self.neg())
        return self.primary()

    def values(self):
        self.take("p", "[")
        out = []
        while self.peek() != ("p", "]"):
            out.append(self.take("v"))
            if self.peek() == ("p", ","):
                self.i += 1
            elif self.peek() != ("p", "]"):
                raise ValueError("filter: expected , or ] in a list")
        self.take("p", "]")
        return out

    def geo(self, kind):
        self.take("p", "(")
        nums, depth = [], 0
        while True:
            tok = self.peek()
            if tok == ("p", "(") or tok == ("p", "["):
                depth += 1
            elif tok == ("p", "]"):
                depth -= 1
            elif tok == ("p", ")"):
                if depth == 0:
                    break
                depth -= 1
            elif tok[0] == "v":
                nums.append(tok[1])
            elif tok != ("p", ","):
                raise ValueError(f"filter: unexpected {tok[1]!r} in a geo filter")
            self.i += 1
        self.take("p", ")")
        if kind == "radius" and len(nums) == 4:
            kind = "radius_resolution"
        elif (kind == "radius" and len(nums) != 3) or (kind == "bbox" and len(nums) != 4):
            raise ValueError(f"filter: wrong number of arguments to a geo filter ({len(nums)})")
        return ("geo", kind, nums)

    def primary(self):
        tok = self.peek()
        if tok == ("p", "("):
            self.i += 1
            e = self.expr()
            self.take("p", ")")
            return e
        if tok[0] == "v" and tok[1] in _GEO and self.peek(1) == ("p", "("):
            self.i += 1
            return self.geo(_GEO[tok[1]])
        field = self.take("v")
        tok = self.peek()
        if tok[0] == "p" and tok[1] in ("=", "!=", ">", ">=", "<", "<="):
            self.i += 1
            return ("cond", field, tok[1], [self.take("v")])
        if tok[0] == "v" and self.peek(1) == ("k", "TO"):
            lo = self.take("v")
            self.i += 1
            return ("cond", field, "TO", [lo, self.take("v")])
        neg = False
        if tok == ("k", "NOT"):
            self.i += 1
            neg = True
        kw = self.take("k")
        if kw == "IN":
            c = ("cond", field, "IN", self.values())
        elif kw == "EXISTS":
            c = ("cond", field, "EXISTS", [])
        elif kw == "CONTAINS":
            c = ("cond", field, "CONTAINS", [self.take("v")])
        elif kw == "STARTS":
            self.take("k", "WITH")
            c = ("cond", field, "STARTS_WITH", [self.take("v")])
        elif kw == "IS" and not neg:
            if self.peek() == ("k", "NOT"):
                self.i += 1
                neg = True
            what = self.take("k")
            if what not in ("NULL", "EMPTY"):
                raise ValueError(f"filter: IS {what}")
            c = ("cond", field, what, [])
        else:
            raise ValueError(f"filter: unexpected {kw!r} after field {field!r}")
        return ("not", c) if neg else c


def parse_filter(s):
    """the FilterCondition tree of a filter string (see the module docstring); ValueError outside the grammar"""
    p = _Parser(s)
    if not p.t:
        raise ValueError("filter: empty expression")
    tree = p.expr()
    if p.i != len(p.t):
        raise ValueError(f"filter: unexpected {p.peek()[1]!r}")
    return tree


_NUM = re.compile(r"[+-]?(?:(?:\d+\.?\d*|\.\d+)(?:[eE][+-]?\d+)?|(?i:inf|infinity|nan))")


def parse_finite_float(raw):
    """Token::parse_finite_float: Rust's f64 syntax, None when it does not parse or is not finite"""
    if not _NUM.fullmatch(raw):
        return None
    x = float(raw)
    return x if x == x and x not in (float("inf"), float("-inf")) else None


def preorder(tree):
    """the nodes of a tree in pre-order (the order of the library's node list)"""
    out = [tree]
    if tree[0] in ("and", "or"):
        for c in tree[1]:
            out += preorder(c)
    elif tree[0] == "not":
        out += preorder(tree[1])
    return out
