"""diffbir.utils.caption (reference utils/caption.py) -> diffbir_b200.utils.caption. LLaVACaptioner is not built."""
from diffbir._unsupported import unsupported
from diffbir_b200.utils.caption import Captioner, EmptyCaptioner, RAMCaptioner  # noqa: F401

LLaVACaptioner = unsupported("LLaVACaptioner", "utils/caption.py:52-145",
                             "use --captioner ram or --captioner none with a --pos_prompt")
