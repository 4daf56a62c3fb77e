"""diffbir.inference (reference inference/__init__.py:1-5) -> diffbir_b200.inference."""
from diffbir_b200.inference import (BFRInferenceLoop, BIDInferenceLoop, BSRInferenceLoop, CustomInferenceLoop,  # noqa: F401
                                    InferenceLoop)

from .._unsupported import unsupported

UnAlignedBFRInferenceLoop = unsupported("UnAlignedBFRInferenceLoop", "inference/unaligned_bfr_loop.py:14-152",
                                        "use diffbir_b200.inference.UnAlignedBFRInferenceLoop, or inference.py "
                                        "--task unaligned_face")
