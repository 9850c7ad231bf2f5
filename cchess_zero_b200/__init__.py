"""cchess_zero_b200 -- batched MCTS self-play engine for Chinese chess on the H100 (sm_90a).

Public surface mirrors the reference's Python API (chengstone/cchess-zero main.py):
GameBoard, MCTS_tree, cchess_main, policy_value_network, plus the batched Engine / SelfPlay drivers."""
from ._lib import EngineError  # noqa: F401

__all__ = ["EngineError", "Engine", "GameBoard", "MCTS_tree", "cchess_main", "policy_value_network"]


def __getattr__(name):
    if name == "Engine":
        from .engine import Engine
        return Engine
    if name == "GameBoard":
        from .rules import GameBoard
        return GameBoard
    if name in ("MCTS_tree", "leaf_node"):
        from . import mcts
        return getattr(mcts, name)
    if name in ("cchess_main", "SelfPlay"):
        from . import selfplay
        return getattr(selfplay, name)
    if name in ("policy_value_network", "policy_value_network_gpus", "PolicyValueNet"):
        from . import net
        return getattr(net, name)
    raise AttributeError(name)
