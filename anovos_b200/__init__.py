"""anovos_b200: H100-native stats_generator / attribute_binning / drift hot path of Anovos."""
__version__ = "0.1.0"

from .frame import ColumnFrame, as_frame  # noqa: E402,F401
