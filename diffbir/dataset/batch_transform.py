"""diffbir.dataset.batch_transform (reference dataset/batch_transform.py) -> diffbir_b200.dataset.batch_transform."""
from diffbir_b200.dataset.batch_transform import BatchTransform, IdentityBatchTransform, RealESRGANBatchTransform  # noqa: F401
