from anovos_b200.data_transformer.transformers import (  # noqa: F401
    IQR_standardization, attribute_binning, boxcox_transformation, cat_to_num_supervised, cat_to_num_transformer,
    cat_to_num_unsupervised, feature_transformation, imputation_MMM, normalization, outlier_categories, z_standardization)
