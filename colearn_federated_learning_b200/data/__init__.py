"""Data layer: Bot-IoT CSV dataset, transforms, federate(), synthetic generators."""
from .datasets import (NetworkTrafficDataset, BaseDataset, ToTensor, ToTensorLong, Normalize,  # noqa: F401
                       FEATURE_COLUMNS, LABEL_COLUMN, CSV_HEADER, CATEGORIES, minmax_scale, xor_toy_dataset,
                       dataset_tensors, category_tensors, category_dataset, DATASET_REGISTRY, register_dataset, load_dataset)
from .synthetic import synthetic_unsw, synthetic_anomaly, synthetic_category, synthetic_images, synthetic_for_model, write_synthetic_csv  # noqa: F401
from .federate import federate, FederatedDataset, FederatedDataLoader, Shard, shard_bounds  # noqa: F401
