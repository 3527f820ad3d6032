"""Import-compatible shim: the batched engine replaces MuJoCo 2.1.0 / mujoco-py on the hot path.  scripts/train_uhc.py imports
`load_model_from_path, MjSim` only under --render; both explain themselves when used."""


def load_model_from_path(path):
    raise NotImplementedError("mujoco_py is replaced by uhc_b200 (libuhc_b200.so); rendering through MuJoCo is not available")


def load_model_from_xml(xml):
    raise NotImplementedError("mujoco_py is replaced by uhc_b200 (libuhc_b200.so)")


class MjSim:
    def __init__(self, model=None):
        raise NotImplementedError("mujoco_py.MjSim is replaced by uhc_b200.engine.Engine")
