"""Real-ESRGAN training-pair synthesis (reference diffbir/dataset): per-sample kernels in numpy, the batch
degradation on the engine (csrc/degrade.cu)."""
