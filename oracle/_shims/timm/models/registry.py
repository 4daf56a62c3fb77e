"""Stand-in for timm.models.registry (imported by ram/models/vit.py)."""


def register_model(fn):
    return fn
