from anovos_b200.data_transformer.transformers import attribute_binning, imputation_MMM  # noqa: F401
