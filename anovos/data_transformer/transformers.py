from anovos_b200.data_transformer.transformers import (  # noqa: F401
    IQR_standardization, attribute_binning, imputation_MMM, normalization, z_standardization)
