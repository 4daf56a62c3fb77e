"""diffbir.dataset.file_backend (reference dataset/file_backend.py) -> diffbir_b200.dataset.file_backend."""
from diffbir_b200.dataset.file_backend import BaseStorageBackend, HardDiskBackend, PetrelBackend  # noqa: F401
