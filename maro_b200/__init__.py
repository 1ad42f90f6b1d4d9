"""maro_b200 — H100-native batched discrete-event simulation core behind MARO's Env / VectorEnv surfaces.

    from maro_b200.simulator import Env
    from maro_b200.vector_env import VectorEnv
    from maro_b200.scenarios.cim.common import Action, ActionType, DecisionEvent
"""
__version__ = "0.1.0"
