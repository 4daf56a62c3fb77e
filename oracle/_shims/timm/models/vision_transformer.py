"""Stand-in for timm.models.vision_transformer (imported by RAM++'s unused ViT backbone, ram/models/vit.py)."""
_cfg = None
PatchEmbed = None
