"""The reference creates a global SparkSession at import (shared/spark.py:97).  The GPU
path has no Spark: callers that do `from anovos.shared.spark import spark` get None."""
spark = sc = sqlContext = None
