#!/usr/bin/env python
"""Generate tests/golden/notebook_monotonic.json from a checkout of anovos/anovos.

    python tests/golden/make_golden_monotonic.py <path of the anovos checkout>

The stored outputs of the two monotonic_binning cells of examples/notebooks/data_transformer__transformers.ipynb (cells 19
and 21, numbered over all cells): the binned columns of the `odf.toPandas().head(5)` frame as displayed, one list of five
values per column (the display shows them as floats: 6.0).  Nothing here executes reference code.
"""
import json
import os
import sys

REF = sys.argv[1] if len(sys.argv) > 1 else "."
OUT = os.path.dirname(os.path.abspath(__file__))
COLUMNS = {19: ["hours-per-week_binned", "education-num_binned"], 21: ["hours-per-week", "education-num"]}


def head_columns(text, names):
    """The values of `names` in the rows 0-4 of a pandas head(5) display, which wraps its columns into blocks."""
    out = {}
    lines = text.splitlines()
    for i, line in enumerate(lines):
        head = line.split()
        if not head or not set(names) & set(head):
            continue
        for k in range(1, 6):
            cells = lines[i + k].split()
            for j, name in enumerate(head):
                if name in names:
                    # a trailing "\" marks a wrapped block; the row label is the first cell
                    out.setdefault(name, []).append(cells[1 + j])
    return {n: [float(v) for v in out[n]] for n in names}


def main():
    nb = json.load(open(REF + "/examples/notebooks/data_transformer__transformers.ipynb"))
    res = []
    for i, c in enumerate(nb["cells"]):
        src = "".join(c["source"])
        if c["cell_type"] != "code" or "monotonic_binning(" not in src:
            continue
        text = "".join("".join(o.get("data", {}).get("text/plain", "")) for o in c.get("outputs", []))
        res.append({"notebook": "transformers", "cell": i, "kind": "head", "source": src,
                    "columns": head_columns(text, COLUMNS[i])})
    json.dump(res, open(OUT + "/notebook_monotonic.json", "w"), indent=0)
    print(len(res), "tables")


if __name__ == "__main__":
    main()
