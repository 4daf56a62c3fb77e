"""CodeformerDataset (reference dataset/codeformer.py) is not built: see diffbir/_unsupported.py."""
from diffbir._unsupported import unsupported

CodeformerDataset = unsupported(
    "dataset.codeformer.CodeformerDataset", "dataset/codeformer.py:21-133",
    "its degradation is per-image cv2 work in dataloader workers with no GPU path; use "
    "diffbir.dataset.realesrgan.RealESRGANDataset with RealESRGANBatchTransform")
