from .sea_raft import *  # noqa: F401,F403
