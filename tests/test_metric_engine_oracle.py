"""CPU: the metric-engine goldens through the oracle's leaf divided on __tsid (labels from each series' first row) and
the row-literal node helpers above it, and the same plans over the leaf divided on the Utf8 labels."""
import pytest

from tests.metric_engine_helpers import _null_first, expected_of, load_metric_engine, oracle_eval, table_batches

G = load_metric_engine()


def _sorted(rows):
    return sorted(rows, key=lambda r: tuple(_null_first(x) for x in r[:-2]) + tuple(r[-2:]))


@pytest.mark.parametrize("case", G["cases"], ids=[c["name"] for c in G["cases"]])
@pytest.mark.parametrize("metric_engine", [True, False], ids=["tsid", "utf8"])
def test_goldens_on_the_cpu(case, metric_engine):
    tags, rows = oracle_eval(case["expr"], G["tables"], case, metric_engine)
    labels = []
    for lab, _, _ in case["expected"]:
        labels += [n for n in lab if n not in labels]
    got = _sorted(tuple(r[tags.index(l)] if l in tags else None for l in labels) + tuple(r[-2:]) for r in rows)
    assert got == expected_of(case, labels)


def test_metric_engine_batches_are_sorted_by_tsid_and_split():
    """The fixture tables as metric-engine batches: sorted by (__tsid, ts), one tsid per label tuple, series cut across
    batches"""
    import pyarrow as pa
    t = G["tables"]["metric_a"]
    batches = table_batches(t, True, splits=3)
    assert len(batches) == 3 and batches[1].schema.names[-1] == "__tsid"
    tab = pa.Table.from_batches(batches)
    ids = tab.column("__tsid").to_pylist()
    ts = tab.column("t").cast(pa.int64()).to_pylist()
    assert list(zip(ids, ts)) == sorted(zip(ids, ts))
    labels = list(zip(*(tab.column(x).to_pylist() for x in t["tags"])))
    assert len(set(zip(ids, labels))) == len(set(ids)) == len(set(labels)) == len(t["series"])
