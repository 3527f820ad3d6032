"""Reward registry (uhc/losses/reward_function.py:823-833).  On the batched engine the imitation reward is fused into the step
kernel (sim_core.h diff_and_reward, restating world_rfc_implicit_reward :12-88 and, with residual_force_mode = explicit,
world_rfc_explicit_reward :253-341, and with reward_id world_rfc_implicit_v1_mul the product form :174-250); the callable keeps the reference signature
`reward(env, state, action, info) -> (reward, c_info[5])` and returns what the kernel computed for the step just taken."""
import numpy as np


def world_rfc_implicit_reward(env, state, action, info):
    return float(env.last_reward), np.asarray(env.last_cinfo, dtype=np.float64)


def world_rfc_explicit_reward(env, state, action, info):
    return float(env.last_reward), np.asarray(env.last_cinfo, dtype=np.float64)


def world_rfc_implicit_v1_mul(env, state, action, info):
    return float(env.last_reward), np.asarray(env.last_cinfo, dtype=np.float64)


reward_func = {"world_rfc_implicit": world_rfc_implicit_reward, "world_rfc_explicit": world_rfc_explicit_reward,
               "world_rfc_implicit_v1_mul": world_rfc_implicit_v1_mul}
