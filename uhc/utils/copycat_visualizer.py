"""Import-compatible shim for scripts/eval_uhc.py --mode vis / disp_stats.  The interactive GL viewer (mujoco-py + glfw) is out of scope
of the batched engine (SURVEY.md section 2 row 17); its render_video output is AgentCopycat.render_motion.  Constructing it explains
what to use instead."""


class CopycatVisualizer:
    def __init__(self, vis_file, agent):
        raise NotImplementedError("interactive visualisation needs mujoco-py/glfw and is not part of the batched engine; "
                                  "run `eval_uhc.py --mode stats` (batched evaluation), or write the evaluation as videos with AgentCopycat.render_motion "
                                  "(the GPU renderer: one mp4 per clip, the simulated humanoid beside the reference motion)")
