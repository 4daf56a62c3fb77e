"""diffbir.dataset.realesrgan (reference dataset/realesrgan.py) -> diffbir_b200.dataset.realesrgan."""
from diffbir_b200.dataset.realesrgan import RealESRGANDataset  # noqa: F401
