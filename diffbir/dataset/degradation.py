"""diffbir.dataset.degradation (reference dataset/degradation.py) -> diffbir_b200.dataset.degradation."""
from diffbir_b200.dataset.degradation import (  # noqa: F401
    bivariate_Gaussian, bivariate_generalized_Gaussian, bivariate_plateau, circular_lowpass_kernel, mesh_grid, pdf2,
    random_add_gaussian_noise_pt, random_add_poisson_noise_pt, random_bivariate_Gaussian,
    random_bivariate_generalized_Gaussian, random_bivariate_plateau, random_mixed_kernels, sigma_matrix2)
