from .plan import BucketPlan, TensorPlan
from .engine import BucketEngine, decode_slot_oracle, engine_oracle, stats_from_slot
from .ddp import DeepReduceDDP
from .comm_hook import DeepReduceHookState, deepreduce_hook, register_deepreduce_hook

__all__ = ["BucketPlan", "TensorPlan", "BucketEngine", "DeepReduceDDP", "DeepReduceHookState", "decode_slot_oracle",
           "deepreduce_hook", "engine_oracle", "register_deepreduce_hook", "stats_from_slot"]
