"""The SMPL body model from the user's own file (include/uhc_mesh.h UhcSmplModel), for Engine.mesh_init.

The model files are licence-gated and do not ship with this project; the reference asks for data/smpl/SMPL_{NEUTRAL,MALE,FEMALE}.pkl
(v1.1.0).  load_smpl_model reads such a .pkl (pickled under Python 2, with or without chumpy objects), the smplx-style .npz with the same
keys, or a directory holding SMPL_NEUTRAL.pkl / .npz.  The pickle comes from outside the program, so it is read through an unpickler that
reconstructs numpy arrays and scipy.sparse matrices only, turns chumpy objects into their array `x`, and refuses every other global: chumpy
itself is not needed."""
import os
import pickle

import numpy as np

NJ, NBETA, NPOSE = 24, 10, 207

_SAFE_GLOBALS = {("numpy.core.multiarray", "_reconstruct"), ("numpy._core.multiarray", "_reconstruct"), ("numpy", "ndarray"),
                  ("numpy", "dtype"), ("numpy.core.multiarray", "scalar"), ("numpy._core.multiarray", "scalar"),
                  # the byte buffers of arrays pickled by Python 3 at protocol <= 2
                  ("_codecs", "encode"),
                  # protocol 0 / 1 objects: object.__new__(cls) for a class that itself passed find_class
                  ("copy_reg", "_reconstructor"), ("copyreg", "_reconstructor"), ("__builtin__", "object"), ("builtins", "object"),
                  # containers in chumpy objects' state
                  ("__builtin__", "set"), ("builtins", "set"), ("__builtin__", "frozenset"), ("builtins", "frozenset")}
_SPARSE_CLASSES = ("csc_matrix", "csr_matrix", "coo_matrix")


class _Chumpy:
    """stands in for any chumpy class: its pickled state's `x` is the array"""

    def __init__(self, *a, **k):
        self.x = None

    def __setstate__(self, state):
        self.x = state.get("x") if isinstance(state, dict) else None


class _Unpickler(pickle.Unpickler):
    def find_class(self, module, name):
        if (module, name) in _SAFE_GLOBALS:
            return super().find_class(module, name)
        if module.split(".")[0] == "scipy" and ".sparse" in module and name in _SPARSE_CLASSES:
            import scipy.sparse
            return getattr(scipy.sparse, name)
        if module == "chumpy" or module.startswith("chumpy."):
            return _Chumpy
        raise pickle.UnpicklingError(f"SMPL model: refusing global {module}.{name}")


def _dense(x):
    if isinstance(x, _Chumpy):
        x = x.x
    if hasattr(x, "toarray"):
        x = x.toarray()
    return np.asarray(x)


def _read(path):
    if os.path.isdir(path):
        for ext in ("pkl", "npz"):
            p = os.path.join(path, "SMPL_NEUTRAL." + ext)
            if os.path.exists(p):
                return _read(p)
        raise FileNotFoundError(os.path.join(path, "SMPL_NEUTRAL.{pkl,npz}"))
    if path.endswith(".npz"):
        with np.load(path, allow_pickle=False) as z:
            return {k: z[k] for k in z.files}
    with open(path, "rb") as f:
        return _Unpickler(f, encoding="latin1").load()


def _as(raw, key, shape):
    if key not in raw:
        raise ValueError(f"SMPL model: missing key {key}")
    try:
        a = _dense(raw[key]).astype(np.float64)
    except (TypeError, ValueError):
        raise ValueError(f"SMPL model: {key} is not a numeric array")
    if a.ndim != len(shape) or any(s is not None and a.shape[i] != s for i, s in enumerate(shape)):
        raise ValueError(f"SMPL model: {key} has shape {a.shape}, expected {tuple('V' if s is None else s for s in shape)}")
    return a


def validate(m):
    """checks a model dict in load_smpl_model's layout: ValueError naming the key at fault"""
    V = m["v_template"].shape[0]
    want = dict(v_template=(V, 3), shapedirs=(V, 3, NBETA), posedirs=(V, 3, NPOSE), J_regressor=(NJ, V), weights=(V, NJ))
    for k, s in want.items():
        if m[k].shape != s:
            raise ValueError(f"SMPL model: {k} has shape {m[k].shape}, expected {s}")
        if not np.isfinite(m[k]).all():
            raise ValueError(f"SMPL model: {k} has non-finite values")
    p = m["parents"]
    if p.shape != (NJ,) or p[0] != -1 or any(not (0 <= p[i] < i) for i in range(1, NJ)):
        raise ValueError("SMPL model: kintree_table / parents: every joint's parent must come before it (parents[i] < i)")
    bad = np.abs(m["weights"].sum(1) - 1.0) > 1e-6
    if bad.any():
        raise ValueError(f"SMPL model: weights of vertex {int(np.argmax(bad))} do not sum to 1")
    if m.get("faces") is not None:
        f = np.asarray(m["faces"])
        if f.ndim != 2 or f.shape[1] != 3 or len(f) < 1 or not (np.issubdtype(f.dtype, np.integer) or (np.isfinite(f).all() and (f == np.round(f)).all())):
            raise ValueError(f"SMPL model: f (the faces) has shape {f.shape}, expected (F, 3) integer vertex indices with F >= 1")
        if f.min() < 0 or f.max() >= V:
            raise ValueError(f"SMPL model: f (the faces) holds a vertex index outside 0 .. {V - 1}")
        m["faces"] = f.astype(np.int32)
    return m


def as_model(model):
    """a model argument as Engine.mesh_init / render_mesh_init take it -- a path (load_smpl_model) or a dict in load_smpl_model's layout, whose
    arrays are checked by validate (a faces value of None, as load_smpl_model returns for a file without `f`, stays absent)"""
    if isinstance(model, (str, os.PathLike)):
        return load_smpl_model(model)
    return validate({k: None if v is None else np.asarray(v) for k, v in model.items()})


def load_smpl_model(path):
    """the SMPL model at `path` (.pkl, .npz, or a directory with SMPL_NEUTRAL.{pkl,npz}) as fp64 arrays: v_template [V][3], shapedirs
    [V][3][10] (the first 10 components, smplx's default num_betas), posedirs [V][3][207], J_regressor [24][V] dense, weights [V][24],
    parents [24] (kintree_table[0] with the root -1), and faces [F][3] int32 when the file has `f` (None otherwise; only mesh rendering needs
    them).  ValueError naming the key for a missing key, inconsistent shapes, parents[i] >= i, non-finite values, a weight row whose sum is
    not 1 within 1e-6, or faces that are not F >= 1 rows of vertex indices in 0 .. V - 1."""
    raw = _read(os.fspath(path))
    if not isinstance(raw, dict):
        raise ValueError("SMPL model: the file does not hold a dict of arrays")
    vt = _as(raw, "v_template", (None, 3))
    V = vt.shape[0]
    sd = _as(raw, "shapedirs", (V, 3, None))
    if sd.shape[2] < NBETA:
        raise ValueError(f"SMPL model: shapedirs has {sd.shape[2]} components, fewer than {NBETA}")
    kt = _as(raw, "kintree_table", (2, NJ))
    parents = kt[0].astype(np.int64)
    parents[0] = -1
    m = dict(v_template=vt, shapedirs=np.ascontiguousarray(sd[:, :, :NBETA]), posedirs=_as(raw, "posedirs", (V, 3, NPOSE)),
             J_regressor=_as(raw, "J_regressor", (NJ, V)), weights=_as(raw, "weights", (V, NJ)), parents=parents.astype(np.int32),
             faces=_dense(raw["f"]) if "f" in raw else None)
    return validate(m)
