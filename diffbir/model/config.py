"""diffbir.model.config (reference model/config.py:1-62): the attention backend is fixed -- the
wgmma flash-attention kernel of libdiffbir_b200.so; there is nothing to select."""


class Config:
    xformers_available = False
    sdp_available = False
    attn_mode = "sm_90a"
