from .craft import *  # noqa: F401,F403
