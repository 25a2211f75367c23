#!/usr/bin/env python
"""Generate tests/golden/notebook_scaling.json from a checkout of anovos/anovos.

    python tests/golden/make_golden_scaling.py <path of the anovos checkout>

The stored Spark outputs of the z_standardization, IQR_standardization and normalization cells of
examples/notebooks/data_transformer__transformers.ipynb: the `describe().show()` tables print_impact printed, in order
(kind "show"; the first table of a cell is "Before", the second "After").  Nothing here executes reference code.
"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden_imputation import show_tables  # noqa: E402

REF = sys.argv[1] if len(sys.argv) > 1 else "."
OUT = os.path.dirname(os.path.abspath(__file__))


def _wanted(src):
    return any(f + "(" in src for f in ("z_standardization", "IQR_standardization", "normalization"))


def main():
    nb = json.load(open(REF + "/examples/notebooks/data_transformer__transformers.ipynb"))
    code = [c for c in nb["cells"] if c["cell_type"] == "code"]
    res = []
    for i, c in enumerate(code):
        src = "".join(c["source"])
        if not _wanted(src):
            continue
        for o in c.get("outputs", []):
            txt = o.get("text")
            if txt:
                for cols, rows in show_tables("".join(txt)):
                    res.append({"notebook": "transformers", "code_cell": i, "kind": "show", "source": src,
                                "columns": cols, "rows": rows})
    json.dump(res, open(OUT + "/notebook_scaling.json", "w"), indent=0)
    print(len(res), "tables")


if __name__ == "__main__":
    main()
