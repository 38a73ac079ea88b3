from .ccmr import *  # noqa: F401,F403
