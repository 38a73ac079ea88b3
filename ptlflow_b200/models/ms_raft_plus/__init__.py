from .ms_raft_plus import *  # noqa: F401,F403
