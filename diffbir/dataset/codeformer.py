"""diffbir.dataset.codeformer (reference dataset/codeformer.py) -> diffbir_b200.dataset.codeformer."""
from diffbir_b200.dataset.codeformer import CodeformerDataset  # noqa: F401
