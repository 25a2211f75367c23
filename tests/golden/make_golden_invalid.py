#!/usr/bin/env python
"""Generate tests/golden/notebook_invalid.json from a checkout of anovos/anovos.

    python tests/golden/make_golden_invalid.py <path of the anovos checkout>

The stored Spark outputs of the invalidEntries_detection cells of examples/notebooks/data_analyzer__quality_checker.ipynb
that are not pandas tables (those are in notebook_quality.json): the `show()` tables of code cells 50-52 (the impact
table and the before / after `describe()` tables).  Cells are cut at the column borders of the `+---+` line, not at
"|" (an invalid_entries cell holds "|"), and only the padding is removed: `show(n, False)` pads on the right and keeps
a value's leading spaces, `show(n)` pads on the left.  Nothing here executes reference code.
"""
import json
import os
import sys

REF = sys.argv[1] if len(sys.argv) > 1 else "."
OUT = os.path.dirname(os.path.abspath(__file__))


def show_tables(text):
    """The `+---+` tables of a cell's text output -> [(columns, rows)], cells cut at the border's '+' positions."""
    out, cur, cuts = [], None, None
    for line in text.splitlines():
        if line.startswith("+"):
            cuts = [i for i, ch in enumerate(line) if ch == "+"]
            continue
        if line.startswith("|") and cuts:
            raw = [line[a + 1:b] for a, b in zip(cuts, cuts[1:])]
            if cur is None:
                left = any(r != r.rstrip() for r in raw)       # a header padded on the right: left-aligned
                cur = ([r.strip() for r in raw], [], left)
                out.append(cur)
            else:
                cur[1].append([r.rstrip() if cur[2] else r.lstrip() for r in raw])
        else:
            cur, cuts = None, None
    return [(c, r) for c, r, _ in out]


def main():
    path = REF + "/examples/notebooks/data_analyzer__quality_checker.ipynb"
    nb = json.load(open(path))
    code = [c for c in nb["cells"] if c["cell_type"] == "code"]
    res = []
    for i, c in enumerate(code):
        src = "".join(c["source"])
        if "invalidEntries_detection(" not in src:
            continue
        text = "".join("".join(o.get("text", "")) for o in c.get("outputs", []))
        for cols, rows in show_tables(text):
            res.append({"notebook": "quality_checker", "code_cell": i, "kind": "show", "source": src, "columns": cols,
                        "rows": rows})
    json.dump(res, open(OUT + "/notebook_invalid.json", "w"), indent=0)
    print(len(res), "tables")


if __name__ == "__main__":
    main()
