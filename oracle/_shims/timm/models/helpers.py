"""Stand-in for timm.models.helpers (imported by RAM++'s unused ViT backbone, ram/models/vit.py)."""
named_apply = None
adapt_input_conv = None
