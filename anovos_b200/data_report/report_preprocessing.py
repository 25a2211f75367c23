"""`save_stats` of anovos.data_report.report_preprocessing (reference /root/reference/src/main/anovos/data_report/
report_preprocessing.py:40-128): the `<master_path>/<function_name>.csv` files through which the stats functions of the
hot path hand their result frames to the report layer (SURVEY.md 8f, row N4).  Only the local / databricks-free file
layout is built: the cloud copies (aws s3 cp / azcopy) and MLflow logging of the reference are control plane."""
from __future__ import annotations

import os

from ..shared.utils import ends_with


def save_stats(spark, idf, master_path, function_name, reread=False, run_type="local", mlflow_config=None, auth_key="NA"):
    """Writes `idf` (a ResultFrame / pandas frame: the output of a measures_of_* / drift / stability function) as
    `<master_path>/<function_name>.csv` with a header row and no index, exactly what `idf.toPandas().to_csv(...,
    index=False)` gives in the reference (:92).  reread=True returns the file read back with inferSchema (:121-127)."""
    if run_type != "local":
        raise NotImplementedError("save_stats: run_type %r (cloud copies are outside the GPU hot-path build)" % run_type)
    local_path = master_path
    if mlflow_config is not None and mlflow_config.get("track_reports", False):
        local_path = local_path + "/" + mlflow_config["run_id"]
    os.makedirs(local_path, exist_ok=True)
    df = idf.toPandas() if hasattr(idf, "toPandas") else idf
    df.to_csv(ends_with(local_path) + function_name + ".csv", index=False)
    if reread:
        from ..data_ingest.data_ingest import read_dataset
        return read_dataset(spark, ends_with(master_path) + function_name + ".csv", "csv", {"header": "True", "inferSchema": "True"})
