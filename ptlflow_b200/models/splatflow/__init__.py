from .splatflow import *  # noqa: F401,F403
