"""invalidEntries_detection against the tables the quality_checker notebook stored (tests/golden/notebook_invalid.json,
code cells 50-52): the `show()` impact tables and the before / after `describe()` counts, for the oracle
(tests/invalid_oracle.py) and for the product's host layer on the NumPy stand-in of anv_flag_members."""
import json
import os

import pytest

import invalid_oracle as O
from test_invalid_cpu import check_print, entry_set, product

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
SHOWN = json.load(open(os.path.join(GOLDEN, "notebook_invalid.json")))

KWARGS = {50: dict(list_of_cols="workclass", detection_type="both", valid_entries=["self-emp.*"],
                   treatment_method="null_replacement"),
          51: dict(list_of_cols=["age", "sex", "race", "workclass", "logfnl"], treatment=True, print_impact=True),
          52: dict(list_of_cols=["sex", "race", "workclass"], treatment=True, output_mode="append", print_impact=True)}


def _tables(cell):
    return [t for t in SHOWN if t["code_cell"] == cell]


def test_golden_holds_the_pins():
    (ex4,) = _tables(50)
    (row,) = ex4["rows"]
    assert row[1] == " State-gov|Local-gov|State-gov|Private|Without-pay|Federal-gov|Never-worked| Private|?"
    assert row[2:] == ["28902", "0.8876"]
    before, after = _tables(51)[1:]
    assert before["rows"][0][:5] == ["count", "32500", "32557", "32247", "32558"]
    assert after["rows"][0][:5] == ["count", "32500", "32548", "32225", "30712"]


def _describe_counts(table, names):
    return {c: table.num_rows - table.column(c).null_count for c in names}


def _check(cell, odf, p):
    show = _tables(cell)[0]
    check_print(p, show)
    if cell == 50:
        assert entry_set(p["invalid_entries"][0]) == entry_set(show["rows"][0][1])
        return
    before, after = _tables(cell)[1:]
    names = before["columns"][1:]
    assert _describe_counts(odf, after["columns"][1:]) == {c: int(v) for c, v in zip(after["columns"][1:], after["rows"][0][1:])}
    assert len(names) == len(after["columns"]) - 1


@pytest.mark.parametrize("cell", [50, 51, 52])
def test_oracle_matches_notebook(income, cell):
    kw = dict(KWARGS[cell])
    kw.pop("print_impact", None)
    odf, p, _ = O.invalidEntries_detection(income, **kw)
    _check(cell, odf, p)
    before = _tables(cell)[1] if cell != 50 else None
    if before is not None:
        names = before["columns"][1:]
        assert _describe_counts(income, names) == {c: int(v) for c, v in zip(names, before["rows"][0][1:])}


@pytest.mark.parametrize("cell", [50, 51, 52])
def test_product_matches_notebook(income, cell):
    odf, p = product(income, **KWARGS[cell])
    _check(cell, odf, p)
