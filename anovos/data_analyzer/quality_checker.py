from anovos_b200.data_analyzer.quality_checker import (  # noqa: F401
    duplicate_detection, nullRows_detection, nullColumns_detection, outlier_detection, IDness_detection,
    biasedness_detection, invalidEntries_detection)
