"""diffbir.dataset.diffjpeg (reference dataset/diffjpeg.py) -> diffbir_b200.dataset.diffjpeg."""
from diffbir_b200.dataset.diffjpeg import DiffJPEG, quality_to_factor  # noqa: F401
