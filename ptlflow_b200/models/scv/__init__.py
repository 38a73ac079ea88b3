from .scv import *  # noqa: F401,F403
