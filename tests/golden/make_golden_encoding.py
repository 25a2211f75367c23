#!/usr/bin/env python
"""Generate tests/golden/notebook_encoding.json from a checkout of anovos/anovos.

    python tests/golden/make_golden_encoding.py <path of the anovos checkout>

The stored Spark outputs of the cat_to_num_unsupervised, cat_to_num_supervised and outlier_categories cells of
examples/notebooks/data_transformer__transformers.ipynb, in order:
  kind "show"    the `show()` tables print_impact printed (summary count / min / max, uniqueValues before / after);
  kind "schema"  the `printSchema()` blocks print_impact printed for one-hot encoding (text after "Before" / "After");
  kind "pandas"  the `toPandas().head(5)` HTML tables (make_golden.notebook_tables).
Nothing here executes reference code.
"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import notebook_tables  # noqa: E402
from make_golden_imputation import show_tables  # noqa: E402

REF = sys.argv[1] if len(sys.argv) > 1 else "."
OUT = os.path.dirname(os.path.abspath(__file__))
FUNCS = ("cat_to_num_unsupervised", "cat_to_num_supervised", "outlier_categories")


def _wanted(src):
    return any(f + "(" in src for f in FUNCS)


def schema_blocks(text):
    """`root` / ` |-- name: type (nullable = ...)` blocks -> [[line, ...]]."""
    out, cur = [], None
    for line in text.splitlines():
        if line == "root":
            cur = []
            out.append(cur)
        elif cur is not None and line.startswith(" |-- "):
            cur.append(line)
        else:
            cur = None
    return out


def main():
    path = REF + "/examples/notebooks/data_transformer__transformers.ipynb"
    nb = json.load(open(path))
    code = [c for c in nb["cells"] if c["cell_type"] == "code"]
    res = []
    for i, c in enumerate(code):
        src = "".join(c["source"])
        if not _wanted(src):
            continue
        text = "".join("".join(o.get("text", "")) for o in c.get("outputs", []))
        for cols, rows in show_tables(text):
            res.append({"notebook": "transformers", "code_cell": i, "kind": "show", "source": src, "columns": cols,
                        "rows": rows})
        for lines in schema_blocks(text):
            res.append({"notebook": "transformers", "code_cell": i, "kind": "schema", "source": src, "lines": lines})
    for t in notebook_tables(path):
        if _wanted(t["source"]):
            res.append({"notebook": "transformers", "code_cell": t["code_cell"], "kind": "pandas", "source": t["source"],
                        "columns": t["columns"], "rows": t["rows"]})
    json.dump(res, open(OUT + "/notebook_encoding.json", "w"), indent=0)
    print(len(res), "tables")


if __name__ == "__main__":
    main()
