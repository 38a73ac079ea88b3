from .raft import *  # noqa: F401,F403  (registers raft, raft_small)
from .gma import *  # noqa: F401,F403  (registers gma)
from .skflow import *  # noqa: F401,F403  (registers skflow)
