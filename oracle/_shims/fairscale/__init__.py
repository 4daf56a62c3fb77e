"""Stand-in for fairscale (only ram/models/vit.py's import of checkpoint_wrapper, unused by RAM++ with Swin-L)."""
