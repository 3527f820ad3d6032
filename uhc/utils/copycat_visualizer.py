"""Import-compatible shim for scripts/eval_uhc.py --mode vis / disp_stats.  The GL viewer (mujoco-py + glfw) is out of scope
of the batched engine (SURVEY.md section 2 row 17); constructing it explains what to use instead."""


class CopycatVisualizer:
    def __init__(self, vis_file, agent):
        raise NotImplementedError("interactive visualisation needs mujoco-py/glfw and is not part of the batched engine; "
                                  "run `eval_uhc.py --mode stats` (batched evaluation) and replay the dumped qpos with the reference viewer")
