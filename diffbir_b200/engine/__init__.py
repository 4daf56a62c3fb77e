"""Kernel-orchestration engines: walk the reference architectures and enqueue the sm_90a
kernels of libdiffbir_b200.so on the current CUDA stream (allocation-free after warm-up, so
every forward is CUDA-graph capturable)."""
