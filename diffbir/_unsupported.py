"""Placeholders for reference names that are outside the accelerated path."""


def unsupported(name: str, reference: str, instead: str):
    """A class called `name` whose constructor raises NotImplementedError (reference file:line cited)."""

    def __init__(self, *args, **kwargs):
        raise NotImplementedError(
            f"diffbir.{name} ({reference}) is not on the H100 hot path (SURVEY.md 8f); {instead}")

    return type(name, (), {"__init__": __init__, "__doc__": f"Not built: {reference}. {instead}",
                           "__module__": "diffbir"})
