"""Stand-in for fairscale.nn.checkpoint.checkpoint_activations (imported by ram/models/vit.py, unused here)."""
checkpoint_wrapper = None
