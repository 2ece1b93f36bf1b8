"""crazyara_b200: H100-native (sm_90a) MCTS + neural-network leaf evaluation engine.

Hot path of QueensGambit/CrazyAra rebuilt as hand-written CUDA behind a C-ABI (include/ara_b200.h).
"""
from ._lib import AraError, LIB_PATH, lib, check  # noqa: F401
