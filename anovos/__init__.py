"""Drop-in module paths of the reference (`anovos.data_analyzer.stats_generator`,
`anovos.drift_stability.drift_detector`, `anovos.data_transformer.transformers`,
`anovos.shared.utils`) re-exporting the CUDA implementation in `anovos_b200`."""
from anovos_b200 import __version__  # noqa: F401
