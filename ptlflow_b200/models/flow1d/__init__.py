from .flow1d import *  # noqa: F401,F403
