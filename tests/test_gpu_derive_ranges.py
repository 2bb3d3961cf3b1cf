"""Term derivation over dictionary prefix ranges: `Index.derive` against `OracleIndex.derive` on small dictionaries built to hit
the edges of the work list (DESIGN.md §3 "Term derivation"): 1- and 2-byte words, empty and non-ASCII first bytes, q[0] == q[1],
matches reachable only through another first byte, the whole-dictionary sweep of 1- and 2-byte terms, ranges across 256-word
tiles, one-word dictionaries and the 150 / 50 caps filled from several ranges at once."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ALPHABET = "abcmnxyz019"
ACCENTED = ["é", "ü", "ж", "日"]  # UTF-8 lead bytes 0xc3, 0xc3, 0xd0, 0xe6


@pytest.fixture(scope="module")
def mb():
    import meilisearch_b200 as m

    m.load_library()
    return m


def _image(words):
    from corpus.pyindexgen import IndexImage

    img = IndexImage(1)
    words = sorted(set(words))
    for i in range(0, len(words), 64):
        img.add_text(i // 64, 0, " ".join(words[i:i + 64]))
    return img.build()


def _check(mb, img, terms):
    from oracle.pyoracle import OracleIndex

    ix, o = mb.Index(img), OracleIndex(img)
    try:
        for max_typo in (1, 2):
            for is_prefix in (0, 1):
                got = ix.derive(terms, [max_typo] * len(terms), [is_prefix] * len(terms))
                for w, (g1, g2) in zip(terms, got):
                    o1, o2 = o.derive(w, max_typo, is_prefix)
                    assert list(g1) == list(o1), (w, max_typo, is_prefix, "one")
                    assert list(g2) == list(o2), (w, max_typo, is_prefix, "two")
    finally:
        ix.close()


def _front_variants(q, letters):
    """words a term reaches only through a first byte other than q[0]"""
    out = [q[1] + q[0] + q[2:], q[1:]]                  # transposition (q1 q0 ...), front deletion (q1 ...)
    for c in letters:
        out += [c + q, c + q[1:]]                        # front insertion (c q0 ...), first-byte substitution (c q1 ...)
    return out


def test_derive_edge_dictionary(mb):
    rng = np.random.default_rng(7)
    words = set()
    for _ in range(2500):  # fills the first-byte ranges well past one 256-word tile
        n = int(rng.integers(3, 9))
        words.add("".join(rng.choice(list(ALPHABET), n)))
    for _ in range(200):
        n = int(rng.integers(2, 6))
        words.add(str(rng.choice(ACCENTED)) + "".join(rng.choice(list(ALPHABET), n)))
    words |= set(ALPHABET) | {"ab", "ba", "aa", "xa", "za", "é", "éa", "aé"}  # 1- and 2-byte words
    bases = ["abcmn", "bacmn", "aabcm", "mmxyz", "xyzab", "éabc", "aébc", "c1a9z"]
    for q in bases:
        words.add(q)
        words.update(_front_variants(q, "bmz9é"))
    # no word starts with "q", "k" or "e": empty first-byte ranges
    img = _image(words)
    terms = bases + ["a", "b", "é", "ab", "ba", "aa", "zz", "xé", "qwerty", "kaaba", "eabcm", "qabcmn", "abcmq", "9zzz",
                     img.word(0), img.word(img.n_words - 1), img.word(img.n_words // 2)]
    terms += [t for q in bases[:4] for t in _front_variants(q, "yq")]
    _check(mb, img, terms)


def test_derive_random_edits(mb):
    rng = np.random.default_rng(11)
    letters = list("abcdefmn") + ACCENTED
    words = {"".join(rng.choice(letters, int(rng.integers(1, 8)))) for _ in range(6000)}
    img = _image(words)
    terms = []
    for _ in range(300):
        w = list(img.word(int(rng.integers(img.n_words))))
        for _ in range(int(rng.integers(3))):
            op, p = int(rng.integers(4)), int(rng.integers(len(w) + 1))
            c = str(rng.choice(letters))
            if op == 0 and p < len(w):
                w[p] = c
            elif op == 1:
                w.insert(p, c)
            elif op == 2 and p < len(w) and len(w) > 1:
                del w[p]
            elif op == 3 and p + 1 < len(w):
                w[p], w[p + 1] = w[p + 1], w[p]
        terms.append("".join(w))
    terms += [t[0] * 2 + t[1:] for t in terms[:40] if len(t) > 1]  # q[0] == q[1]
    _check(mb, img, terms)


def test_derive_one_word_dictionary(mb):
    img = _image(["hello"])
    _check(mb, img, ["hello", "hallo", "ehllo", "xhello", "ello", "helo", "h", "he", "hx", "zzzzz"])


def test_derive_caps_across_ranges(mb):
    # one term whose matches fill both caps from its own first byte and from every other range family, interleaved in word-id order
    q = "mnopqrst"
    subs = "abcdefghijklmnopqrstuvwxyz0123456789"
    words = set()
    for p in range(1, len(q)):
        for c in subs:
            words.add(q[:p] + c + q[p + 1:])               # same first byte, d <= 1
            words.add(q[:p] + c + q[p:])
    for c in subs:
        if c not in "mn":
            words.add(c + q[1:])                          # (c q1 ...)
            words.add(c + q)                              # (c q0 ...)
    words.update([q[1] + q[0] + q[2:], q[1:], q[1:] + "a"])
    img = _image(words)
    _check(mb, img, [q, "nmopqrst", "xnopqrst", "mnopqrsx", "mmopqrst"])
