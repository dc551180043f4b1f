"""CPU: the label_replace regex engine through the built library, no device needed.  Every regex and replacement of the
reference's label.result; a differential test against Python's `re.fullmatch(.., re.DOTALL)` (leftmost-first over
code points, as Rust's `regex`) on seeded patterns from the supported grammar over ASCII and multibyte inputs; Rust's
verdict on a table of patterns; the replacement's `$` expansion edge cases; the destination label name check."""
import json
import os
import random
import re

import pytest

from greptimedb_b200 import B2PError
from greptimedb_b200.plan import (REGEX_INVALID, REGEX_OK, REGEX_UNSUPPORTED, label_regex_check,
                                  label_regex_replace)

GOLDEN = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "reference_label_vectors.json")))


def test_golden_regexes_and_replacements():
    """label_replace(test{host=..}, dst, replacement, "idc", regex) of the goldens, value by value"""
    seen = 0
    for c in GOLDEN["cases"]:
        m = re.fullmatch(r'label_replace\(test\{host="host\d"\}, "([^"]*)", "([^"]*)", "idc", "([^"]*)"\)( == .*)?', c["query"])
        if not m or not c["rows"] or m.group(3) == "" or m.group(1) == "idc":
            continue
        dst, rep, rx = m.group(1), m.group(2), m.group(3)
        i_dst, i_idc = c["columns"].index(dst), c["columns"].index("idc")
        for row in c["rows"]:
            assert label_regex_replace(rx, rep, row[i_idc]) == row[i_dst], (rx, row)
            seen += 1
    assert seen == 34


VERDICTS = {
    REGEX_OK: ["", "(.*):(.*)", "idc2.*", "(.*)-[^-]+", "a|", "()", "(?:)", "[]a]", "[^]a]", "[a-]", "[-a]",
               "[[:alpha:]][[:^digit:]]", r"\x41\x{1F600}\n\t\.\$", "(?P<n>a)(?<m>b)", "a{2}", "a{2,}", "a{2,3}?",
               "(?s).", "(?-s:.)", "(?m)^a$", "(?U)a+", r"\Aa\z", "é+", "[α-ω]"],
    REGEX_INVALID: ["(?=a)", "(?!a)", "(?<=a)", "(?<!a)", r"\1", r"\0", "(.*", "a)", "a{2,1}", "*a", "+", "a|*", "[a",
                    "[z-a]", r"\Z", r"\e", "(?P=n)", "(?P<n>a)(?P<n>b)", "(?<>a)", "(?)", "(?-)", "(?ss)", "(?q)",
                    "[[:nope:]]", r"\x4", r"\x{110000}", "\\"],
    REGEX_UNSUPPORTED: [r"\d", r"\w", r"\s", r"\b", r"\B", r"\pL", r"\p{Greek}", "(?i)a", "(?x)a", "(?-u)a", "a**",
                        "^*", "a{1001}", "a{,3}", "a{x}", "[a[b]]", "[a&&b]", "[a--b]", r"\!", "(?P<é>a)",
                        "(((((((((((((((((((((((((((((((((((((((((((((((((((((((((((((((((((a)))))))))))))))))))))))))"
                        "))))))))))))))))))))))))))))))))))))))))))", "(a{1000}){30}"],
}


@pytest.mark.parametrize("verdict", sorted(VERDICTS))
def test_verdicts(verdict):
    for p in VERDICTS[verdict]:
        assert label_regex_check(p) == verdict, p
        if verdict != REGEX_OK:
            with pytest.raises(B2PError):
                label_regex_replace(p, "", "a")


@pytest.mark.parametrize("rx,rep,value,want", [
    ("(a)(b)?", "$1a", "a", ""),            # $1a names group "1a"
    ("(a)(b)?", "${1}a", "a", "aa"),
    ("(a)(b)?", "$$", "a", "$"),
    ("(a)(b)?", "[$2]", "a", "[]"),          # did not take part
    ("(a)(b)?", "[$9|${x}]", "a", "[|]"),    # does not exist
    ("(a)(b)?", r"\1-\2-\\", "ab", "a-b-"),  # \N is ${N}; a bare backslash is ${}
    ("(a)", "$", "a", "$"),
    ("(a)", "${1", "a", "${1"),
    ("(a)", "${+1}", "a", "a"),              # usize::from_str takes a sign
    ("(?P<w>a+)(?<x>b)", "$w:${x}:$0", "aab", "aa:b:aab"),
    ("b", "x", "abc", "abc"),                # no match: the value unchanged
    ("", "x", "", "x"),
    ("(a*)*", "<$1>", "aa", "<aa>"),        # the Pike VM's answer for a nested empty loop (Rust's too)
    ("(a*)+", "<$1>", "aa", "<aa>"),
    ("(a|ab)(c|bcd)(d*)", "$1|$2|$3", "abcd", "a|bcd|"),
    ("(?U)(a+)(a*)", "$1|$2", "aaa", "a|aa"),
    ("(?m)a$\nb", "ok", "a\nb", "ok"),
    ("a$", "ok", "a\n", "a\n"),              # `$` is the end of the text only (not before a final \n)
    ("(.)(.)", "$2$1", "é€", "€é"),
    ("[^a]", "x", "\n", "x"),
])
def test_replacement_edges(rx, rep, value, want):
    assert label_regex_replace(rx, rep, value) == want


# ---- differential against Python's re --------------------------------------------------------------------------------
ALPHABET = ["a", "b", "c", "-", ":", "é", "€", "😀", "\n", "."]


def gen(rng, depth=0):
    """(rust pattern, python pattern) from the supported grammar, without nested empty-matching repetitions"""
    k = rng.randrange(9 if depth < 3 else 4)
    if k == 0:
        ch = rng.choice(ALPHABET)
        return (re.escape(ch) if ch in ".-" else ch.replace("\n", r"\n"),) * 2
    if k == 1:
        return (".", ".")
    if k == 2:
        neg = rng.random() < 0.3
        items = rng.sample(["a", "b-c", "é", "€-😀", r"\n", ":"], rng.randrange(1, 4))
        body = ("^" if neg else "") + "".join(items)
        return (f"[{body}]",) * 2
    if k == 3:
        if rng.random() < 0.5:
            return ("[[:alpha:]]", "[A-Za-z]")
        return ("[[:^alpha:]]", "[^A-Za-z]")
    if k in (4, 5):
        parts = [gen(rng, depth + 1) for _ in range(rng.randrange(1, 4))]
        return "".join(p[0] for p in parts), "".join(p[1] for p in parts)
    if k == 6:
        a, b = gen(rng, depth + 1), gen(rng, depth + 1)
        return f"{a[0]}|{b[0]}", f"{a[1]}|{b[1]}"
    if k == 7:
        a = gen(rng, depth + 1)
        kind = rng.randrange(4)
        if kind == 0:
            return f"({a[0]})", f"({a[1]})"
        if kind == 1:
            return f"(?:{a[0]})", f"(?:{a[1]})"
        name = f"g{rng.randrange(1000)}_{depth}"
        return f"(?<{name}>{a[0]})" if kind == 2 else f"(?P<{name}>{a[0]})", f"(?P<{name}>{a[1]})"
    a = gen(rng, depth + 1)
    if re.fullmatch(a[1], "", re.DOTALL):  # an empty-matching body under a loop: excluded (see the edge table)
        return a
    q = rng.choice(["*", "+", "?", "{2}", "{1,3}", "{0,}", "{2,}"]) + rng.choice(["", "?"])
    return f"(?:{a[0]}){q}", f"(?:{a[1]}){q}"


def inputs(rng):
    return ["".join(rng.choice(ALPHABET) for _ in range(rng.randrange(0, 8))) for _ in range(6)]


def test_differential_against_python_re():
    rng = random.Random(0x1ABE1)
    checked = 0
    for _ in range(3000):
        rs, py = gen(rng)
        # duplicate names are an error in both; skip them
        names = re.findall(r"\?P?<(\w+)>", rs)
        if len(names) != len(set(names)):
            continue
        assert label_regex_check(rs) == REGEX_OK, rs
        cpy = re.compile(py, re.DOTALL)
        n_groups = cpy.groups
        rep = "|".join(f"${{{i}}}" for i in range(n_groups + 1))
        vals = inputs(rng)
        # values the pattern matches, built from a Python match of a random string, are rare: add some via sampling
        for v in vals:
            m = cpy.fullmatch(v)
            want = v if m is None else "|".join(m.group(i) or "" for i in range(n_groups + 1))
            assert label_regex_replace(rs, rep, v) == want, (rs, v)
            checked += 1
    assert checked > 15000


def test_differential_on_matching_inputs():
    """inputs drawn so that they match: each pattern run on strings Python's re accepts"""
    rng = random.Random(7)
    hits = 0
    for _ in range(3000):
        rs, py = gen(rng)
        names = re.findall(r"\?P?<(\w+)>", rs)
        if len(names) != len(set(names)):
            continue
        cpy = re.compile(py, re.DOTALL)
        rep = "|".join(f"${{{i}}}" for i in range(cpy.groups + 1))
        for _ in range(40):
            v = "".join(rng.choice(ALPHABET) for _ in range(rng.randrange(0, 5)))
            m = cpy.fullmatch(v)
            if m is None:
                continue
            assert label_regex_replace(rs, rep, v) == "|".join(m.group(i) or "" for i in range(cpy.groups + 1)), (rs, v)
            hits += 1
    assert hits > 2000


@pytest.mark.parametrize("name,ok", [("new_idc", True), ("_a9", True), ("A", True), ("~invalid", False), ("", False),
                                     ("__name__", False), ("__x", False), ("9a", False), ("a-b", False), ("é", False)])
def test_destination_label_name(name, ok):
    """validate_label_name, checked at create before the regex and the child (which may be NULL for that)"""
    from greptimedb_b200 import _lib
    L = _lib.load()
    assert not L.b2p_plan_label_replace_create(None, None, name.encode(), b"", b"", b"(")
    msg = L.b2p_plan_last_error().decode()
    if ok:
        assert msg == "Invalid regular expression in label_replace(): (", name
    else:
        assert msg == f"Invalid destination label name in label_replace(): {name}", name
