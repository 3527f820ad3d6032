"""Import-compatible shim (scripts/train_uhc.py:72 under --render)."""


class MjViewer:
    def __init__(self, sim=None):
        raise NotImplementedError("MjViewer (GL rendering) is not part of the batched engine")
