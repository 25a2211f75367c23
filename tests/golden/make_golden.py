#!/usr/bin/env python
"""Generate the golden fixtures under tests/golden/ from a checkout of anovos/anovos.

    python tests/golden/make_golden.py <path of the anovos checkout>

The outputs are committed, so the tests never need the checkout.  Nothing here executes reference code
(it needs a JVM + Spark, absent here): the vectors are the REAL Spark outputs the
reference stores in its notebooks, plus the input datasets they were computed on.

  income.parquet          examples/data/income_dataset/csv (minus dt_1, dt_2, as the
                          notebooks do), typed like Spark's CSV inferSchema
  income_source.parquet   examples/data/income_dataset/source/sample1.csv (drift source)
  income_part1.parquet    data/test_dataset/part-00001-*.snappy.parquet (test_transformers.py:22)
  income_part0.parquet    data/test_dataset/part-00000-*.snappy.parquet (test_association_evaluator.py:17)
  stability.parquet       examples/data/income_dataset/stability_index/{0..11} stacked, column `_ds` = dataset id
  income_partitions.json  how Spark split the income CSV when the notebooks ran: Hadoop line splits of the 5.9 MB file at
                          spark.sql.files.openCostInBytes = 4 MiB (any local[*] with >= 3 cores) -> rows per partition
  notebook_stats.json     stored outputs of examples/notebooks/data_analyzer__stats_generator.ipynb
  notebook_drift.json     stored outputs of examples/notebooks/drift_stability.ipynb
  notebook_quality.json   stored outputs of examples/notebooks/data_analyzer__quality_checker.ipynb
  notebook_association.json  stored outputs of examples/notebooks/data_analyzer__association_evaluator.ipynb
"""
import html.parser
import json
import os
import shutil
import sys

import pyarrow as pa
import pyarrow.csv as pacsv
import pyarrow.parquet as pq

REF = sys.argv[1] if len(sys.argv) > 1 else "."
OUT = os.path.dirname(os.path.abspath(__file__))

INT_COLS = ["age", "fnlwgt", "education-num", "capital-gain", "capital-loss", "hours-per-week", "dupl_age"]
DBL_COLS = ["logfnl", "latitude", "longitude"]


def read_income(path):
    hdr = open(path).readline().strip().split(",")
    types = {}
    for c in hdr:
        if c in INT_COLS:
            types[c] = pa.int32()
        elif c in DBL_COLS:
            types[c] = pa.float64()
        else:
            types[c] = pa.string()
    t = pacsv.read_csv(path, convert_options=pacsv.ConvertOptions(
        column_types=types, strings_can_be_null=True, null_values=[""]))
    return t.drop_columns([c for c in ("dt_1", "dt_2") if c in t.column_names])


class _Tables(html.parser.HTMLParser):
    def __init__(self):
        super().__init__()
        self.tables, self._row, self._cell, self._in = [], None, None, False

    def handle_starttag(self, tag, attrs):
        if tag == "table":
            self.tables.append([])
        elif tag == "tr":
            self._row = []
        elif tag in ("td", "th"):
            self._cell = ""
            self._in = True

    def handle_endtag(self, tag):
        if tag in ("td", "th"):
            self._row.append(self._cell.strip())
            self._in = False
        elif tag == "tr" and self._row is not None:
            self.tables[-1].append(self._row)
            self._row = None

    def handle_data(self, data):
        if self._in:
            self._cell += data


def notebook_tables(path):
    nb = json.load(open(path))
    out = []
    code = [c for c in nb["cells"] if c["cell_type"] == "code"]
    for i, c in enumerate(code):
        for o in c.get("outputs", []):
            h = o.get("data", {}).get("text/html")
            if not h:
                continue
            p = _Tables()
            p.feed("".join(h))
            for t in p.tables:
                header = t[0][1:]
                rows = [r[1:] for r in t[1:]]
                out.append({"code_cell": i, "source": "".join(c["source"]), "columns": header, "rows": rows})
    return out


def csv_partition_rows(path, split_bytes=4 * 1024 * 1024):
    """Rows per Spark partition of a single CSV: FilePartition cuts the file every maxSplitBytes = max(openCostInBytes,
    min(maxPartitionBytes, totalBytes / cores)) = 4 MiB here; Hadoop's LineRecordReader gives a split every line that
    STARTS at an offset <= its end (and skips its own first, partial line)."""
    raw = open(path, "rb").read()
    starts, pos = [], 0
    for line in raw.split(b"\n")[:-1] if raw.endswith(b"\n") else raw.split(b"\n"):
        starts.append(pos)
        pos += len(line) + 1
    starts = starts[1:]                                   # header line
    rows, end = [], split_bytes
    while True:
        k = sum(1 for s_ in starts if s_ <= end) - sum(rows)
        rows.append(k)
        if end >= len(raw):
            break
        end += split_bytes
    return {"file_bytes": len(raw), "split_bytes": split_bytes, "rows_per_partition": [r for r in rows if r]}


def main():
    inc = read_income(REF + "/examples/data/income_dataset/csv/part-00000-8beb3930-8a44-4b7b-906b-a6deca466d9f-c000.csv")
    pq.write_table(inc, OUT + "/income.parquet", compression="zstd")
    src = read_income(REF + "/examples/data/income_dataset/source/sample1.csv")
    pq.write_table(src, OUT + "/income_source.parquet", compression="zstd")
    shutil.copyfile(REF + "/data/test_dataset/part-00001-3eb0f7bb-05c2-46ec-8913-23ba231d2734-c000.snappy.parquet",
                    OUT + "/income_part1.parquet")
    os.chmod(OUT + "/income_part1.parquet", 0o644)
    shutil.copyfile(REF + "/data/test_dataset/part-00000-3eb0f7bb-05c2-46ec-8913-23ba231d2734-c000.snappy.parquet",
                    OUT + "/income_part0.parquet")   # test_association_evaluator.py:17, test_quality_checker.py:16
    os.chmod(OUT + "/income_part0.parquet", 0o644)
    parts = []
    for ds in range(12):
        d = REF + "/examples/data/income_dataset/stability_index/%d" % ds
        f = [x for x in os.listdir(d) if x.endswith(".csv")][0]
        t = pacsv.read_csv(os.path.join(d, f))
        parts.append(t.append_column("_ds", pa.array([ds] * t.num_rows, pa.int32())))
    pq.write_table(pa.concat_tables(parts, promote_options="default"), OUT + "/stability.parquet", compression="zstd")
    json.dump(notebook_tables(REF + "/examples/notebooks/data_analyzer__stats_generator.ipynb"),
              open(OUT + "/notebook_stats.json", "w"), indent=0)
    json.dump(notebook_tables(REF + "/examples/notebooks/drift_stability.ipynb"),
              open(OUT + "/notebook_drift.json", "w"), indent=0)
    json.dump(notebook_tables(REF + "/examples/notebooks/data_analyzer__quality_checker.ipynb"),
              open(OUT + "/notebook_quality.json", "w"), indent=0)
    json.dump(notebook_tables(REF + "/examples/notebooks/data_analyzer__association_evaluator.ipynb"),
              open(OUT + "/notebook_association.json", "w"), indent=0)
    json.dump(csv_partition_rows(REF + "/examples/data/income_dataset/csv/part-00000-8beb3930-8a44-4b7b-906b-a6deca466d9f-c000.csv"),
              open(OUT + "/income_partitions.json", "w"))
    print(inc.schema, inc.num_rows, src.num_rows)


if __name__ == "__main__":
    main()
