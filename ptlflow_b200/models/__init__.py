from .raft import *  # noqa: F401,F403  (registers raft, raft_small)
from .gma import *  # noqa: F401,F403  (registers gma)
from .skflow import *  # noqa: F401,F403  (registers skflow)
from .sea_raft import *  # noqa: F401,F403  (registers sea_raft, sea_raft_s, sea_raft_m, sea_raft_l)
