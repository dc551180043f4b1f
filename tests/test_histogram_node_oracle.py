"""CPU: the histogram_quantile-over-any-child restatement (tests/histogram_node_oracle.py) reproduces the reference's
printed tables, and sorts its input as HistogramFold requires."""
import json
import math
import os

import pytest

from tests import histogram_node_oracle as hno
from tests.helpers import GOLDEN_DIR
from tests.topk_oracle import topk_rows

with open(os.path.join(GOLDEN_DIR, "reference_histogram_node_vectors.json")) as f:
    G = json.load(f)
CASES = {c["name"]: c for c in G["cases"]}


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_reproduces_the_golden_tables(name):
    c = CASES[name]
    rows, tags = hno.golden_child_rows(G["tables"][c["table"]], c)
    got, names = hno.histogram_node(rows, tags, float(c["phi"]))
    if "outer" in c:
        got = topk_rows(False, c["outer"]["k"], got, names)
    assert len(got) == len(c["expected"]), name
    for (v, lab, ts), (e_lab, e_ts, e_v) in zip(sorted(got, key=lambda r: (sorted(r[1].items()), r[2])) if "outer" not in c
                                                else got, c["expected"]):
        assert lab == e_lab and ts == e_ts and (repr(v) == repr(float(e_v)) or math.isnan(v) and e_v == "NaN"), (name, v, e_v)


def test_no_le_tag_is_an_empty_result():
    rows = [(1.0, {"job": "a"}, 0), (2.0, {"job": "b"}, 0)]
    assert hno.histogram_node(rows, ["job"], 0.5) == ([], [])


def test_input_is_sorted_by_tags_ts_and_numeric_le():
    """Rows in any order fold as the sorted input: the other tags with NULL last, ts, then le as a number with
    unparsable and NULL bounds after +Inf."""
    rows = [(10.0, {"le": "+Inf", "s": "a"}, 0), (4.0, {"le": "1e0", "s": "a"}, 0), (2.0, {"le": ".5", "s": "a"}, 0),
            (8.0, {"le": "+Inf", "s": None}, 0), (8.0, {"le": "10", "s": None}, 0), (1.0, {"le": "0.1", "s": None}, 0)]
    got, names = hno.histogram_node(rows, ["le", "s"], 0.5)
    assert names == ["s"]
    assert [(lab["s"], ts) for _, lab, ts in got] == [("a", 0), (None, 0)]
    # a: buckets (0.5, 2), (1, 4), (+Inf, 10): rank 5 falls in +Inf, so the last finite bound
    assert got[0][0] == 1.0
    # NULL: (0.1, 1), (10, 8), (+Inf, 8): rank 4 in (0.1, 10]
    assert got[1][0] == 0.1 + (10 - 0.1) / (8 - 1) * (4 - 1)
