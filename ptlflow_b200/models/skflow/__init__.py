from .skflow import skflow  # noqa: F401
