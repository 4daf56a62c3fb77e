"""Storage backends of the dataset (reference dataset/file_backend.py)."""
from abc import ABCMeta, abstractmethod
from pathlib import Path
from typing import Union


class BaseStorageBackend(metaclass=ABCMeta):
    """A backend returns a file's bytes for a path."""

    @property
    def name(self) -> str:
        return type(self).__name__

    @abstractmethod
    def get(self, filepath: str) -> bytes:
        ...


class HardDiskBackend(BaseStorageBackend):
    """Reads files from the local file system."""

    def get(self, filepath: Union[str, Path]) -> bytes:
        return Path(filepath).read_bytes()


class PetrelBackend(BaseStorageBackend):
    def __init__(self, *args, **kwargs):
        raise NotImplementedError("PetrelBackend (reference dataset/file_backend.py) needs petrel_client, a "
                                  "cluster-specific storage client; use HardDiskBackend")

    def get(self, filepath):
        raise NotImplementedError
