from .llaflow import *  # noqa: F401,F403
