import json
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def income():
    import pyarrow.parquet as pq
    return pq.read_table(os.path.join(GOLDEN, "income.parquet"))


@pytest.fixture(scope="session")
def income_source():
    import pyarrow.parquet as pq
    return pq.read_table(os.path.join(GOLDEN, "income_source.parquet"))


@pytest.fixture(scope="session")
def income_part0():
    import pyarrow.parquet as pq
    return pq.read_table(os.path.join(GOLDEN, "income_part0.parquet"))


@pytest.fixture(scope="session")
def income_part1():
    import pyarrow.parquet as pq
    return pq.read_table(os.path.join(GOLDEN, "income_part1.parquet"))


def _tables(name):
    return json.load(open(os.path.join(GOLDEN, name)))


@pytest.fixture(scope="session")
def nb_stats():
    """code_cell index -> table dict of the stats_generator notebook."""
    return {t["code_cell"]: t for t in _tables("notebook_stats.json")}


@pytest.fixture(scope="session")
def nb_quality():
    return {t["code_cell"]: t for t in _tables("notebook_quality.json")}


@pytest.fixture(scope="session")
def nb_assoc():
    return {t["code_cell"]: t for t in _tables("notebook_association.json")}


@pytest.fixture(scope="session")
def income_spark(income):
    """The income table tagged with the scan partitions Spark used when the reference notebooks ran."""
    import json
    from oracle import api as O
    return O.with_spark_partitions(income, json.load(open(os.path.join(GOLDEN, "income_partitions.json")))["rows_per_partition"])


@pytest.fixture(scope="session")
def nb_drift():
    return {t["code_cell"]: t for t in _tables("notebook_drift.json")}
