#!/usr/bin/env python
"""Generate tests/golden/notebook_transform.json from a checkout of anovos/anovos.

    python tests/golden/make_golden_transform.py <path of the anovos checkout>

The stored Spark outputs of the feature_transformation and boxcox_transformation cells of
examples/notebooks/data_transformer__transformers.ipynb (cells 108-112 and 115-116, numbered over all cells): the
`describe().show()` tables print_impact printed, in order (kind "show"; the first table of a cell is "Before", the second
"After"), and the "Best BoxCox Parameter(s)" list of the Box-Cox cells (kind "lambdas").  Nothing here executes
reference code.
"""
import json
import os
import re
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden_imputation import show_tables  # noqa: E402

REF = sys.argv[1] if len(sys.argv) > 1 else "."
OUT = os.path.dirname(os.path.abspath(__file__))


def main():
    nb = json.load(open(REF + "/examples/notebooks/data_transformer__transformers.ipynb"))
    res = []
    for i, c in enumerate(nb["cells"]):
        src = "".join(c["source"])
        if c["cell_type"] != "code" or not ("feature_transformation(" in src or "boxcox_transformation(" in src):
            continue
        for o in c.get("outputs", []):
            txt = "".join(o.get("text", ""))
            if not txt:
                continue
            m = re.search(r"Best BoxCox Parameter\(s\):\s*(\[.*\])", txt)
            if m:
                res.append({"notebook": "transformers", "cell": i, "kind": "lambdas", "source": src,
                            "lambdas": json.loads(m.group(1))})
            for cols, rows in show_tables(txt):
                res.append({"notebook": "transformers", "cell": i, "kind": "show", "source": src, "columns": cols,
                            "rows": rows})
    json.dump(res, open(OUT + "/notebook_transform.json", "w"), indent=0)
    print(len(res), "tables")


if __name__ == "__main__":
    main()
