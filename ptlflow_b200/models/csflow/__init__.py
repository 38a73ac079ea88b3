from .csflow import *  # noqa: F401,F403
