#!/usr/bin/env python
"""Generate tests/golden/notebook_imputation.json from a checkout of anovos/anovos.

    python tests/golden/make_golden_imputation.py <path of the anovos checkout>

The stored Spark outputs of the imputation_MMM cells of examples/notebooks/data_transformer__transformers.ipynb and of the
nullColumns_detection(treatment_method="MMM") cells of examples/notebooks/data_analyzer__quality_checker.ipynb: the text
tables `show()` printed (kind "show") and the pandas tables `toPandas().head()` rendered (kind "pandas").  Nothing here
executes reference code.
"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import notebook_tables  # noqa: E402

REF = sys.argv[1] if len(sys.argv) > 1 else "."
OUT = os.path.dirname(os.path.abspath(__file__))


def _wanted(src):
    return "imputation_MMM(" in src or ("nullColumns_detection(" in src and "MMM" in src)


def show_tables(text):
    """The `+---+` tables of a cell's text output -> [(columns, rows)]."""
    out, cur = [], None
    for line in text.splitlines():
        if line.startswith("+"):
            continue
        if line.startswith("|"):
            cells = [c.strip() for c in line.strip().strip("|").split("|")]
            if cur is None:
                cur = (cells, [])
                out.append(cur)
            else:
                cur[1].append(cells)
        else:
            cur = None
    return out


def extract(path, notebook):
    nb = json.load(open(path))
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
                    res.append({"notebook": notebook, "code_cell": i, "kind": "show", "source": src, "columns": cols,
                                "rows": rows})
    for t in notebook_tables(path):
        if _wanted(t["source"]):
            res.append(dict(t, notebook=notebook, kind="pandas"))
    return res


def main():
    tabs = extract(REF + "/examples/notebooks/data_transformer__transformers.ipynb", "transformers")
    tabs += extract(REF + "/examples/notebooks/data_analyzer__quality_checker.ipynb", "quality_checker")
    json.dump(tabs, open(OUT + "/notebook_imputation.json", "w"), indent=0)
    print(len(tabs), "tables")


if __name__ == "__main__":
    main()
