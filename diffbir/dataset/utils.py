"""diffbir.dataset.utils (reference dataset/utils.py) -> diffbir_b200.dataset.utils."""
from diffbir_b200.dataset.utils import DiffJPEG, USMSharp, augment, center_crop_arr, filter2D, load_file_list, load_file_metas, random_crop_arr  # noqa: F401
