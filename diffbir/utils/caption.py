"""diffbir.utils.caption (reference utils/caption.py) -> diffbir_b200.utils.caption."""
from diffbir_b200.utils.caption import Captioner, EmptyCaptioner, LLaVACaptioner, RAMCaptioner  # noqa: F401
