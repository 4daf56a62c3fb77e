"""diffbir.dataset (reference dataset/) -> diffbir_b200.dataset."""
