"""Stand-in for timm.models.hub: RAM++'s checkpoint helpers import download_cached_file; the fixture generator
never downloads."""


def download_cached_file(*args, **kwargs):
    raise RuntimeError("no network: the fixture generators never download checkpoints")
