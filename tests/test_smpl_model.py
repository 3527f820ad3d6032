"""CPU: uhc_b200.smpl_model.load_smpl_model reads the SMPL model in its three forms and refuses malformed files and foreign pickles."""
import io
import os
import pickle
import sys
import types

import numpy as np
import pytest
import scipy.sparse

from uhc_b200.smpl_model import load_smpl_model

PARENTS = [-1, 0, 0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 9, 9, 12, 13, 14, 16, 17, 18, 19, 20, 21]


def synthetic(V=40, seed=0, nbeta=10):
    rng = np.random.RandomState(seed)
    w = rng.rand(V, 24) * (rng.rand(V, 24) < 0.2)
    w[np.arange(V), rng.randint(0, 24, V)] += 1.0
    w /= w.sum(1, keepdims=True)
    kt = np.array([[4294967295] + PARENTS[1:], list(range(24))], np.int64)
    return dict(v_template=rng.normal(0, 0.3, (V, 3)), shapedirs=rng.normal(0, 0.01, (V, 3, nbeta)), posedirs=rng.normal(0, 0.01, (V, 3, 207)),
                J_regressor=rng.dirichlet(np.ones(V), 24), weights=w, kintree_table=kt, f=rng.randint(0, V, (10, 3)))


def _check(m, raw):
    assert m["v_template"].dtype == np.float64 and m["v_template"].shape == raw["v_template"].shape
    assert np.array_equal(m["v_template"], raw["v_template"]) and np.array_equal(m["shapedirs"], raw["shapedirs"][:, :, :10])
    assert np.array_equal(m["posedirs"], raw["posedirs"]) and np.array_equal(m["weights"], raw["weights"])
    assert np.array_equal(m["J_regressor"], np.asarray(raw["J_regressor"].toarray() if hasattr(raw["J_regressor"], "toarray") else raw["J_regressor"]))
    assert list(m["parents"]) == PARENTS


def test_npz_and_directory(tmp_path):
    raw = synthetic(nbeta=300)
    np.savez(tmp_path / "SMPL_NEUTRAL.npz", **raw)
    _check(load_smpl_model(str(tmp_path / "SMPL_NEUTRAL.npz")), raw)
    _check(load_smpl_model(str(tmp_path)), raw)
    with pytest.raises(FileNotFoundError):
        load_smpl_model(str(tmp_path / "nowhere"))


def test_pickle_with_chumpy_objects_loads_without_chumpy(tmp_path):
    """written while a stand-in chumpy.ch.Ch is importable, read after it is gone: the loader needs no chumpy"""
    raw = synthetic()
    raw["J_regressor"] = scipy.sparse.csc_matrix(raw["J_regressor"])

    class Ch:
        def __init__(self, x):
            self.x = x

        def __getstate__(self):
            return {"x": self.x, "_dirty_vars": set()}

    mods = {"chumpy": types.ModuleType("chumpy"), "chumpy.ch": types.ModuleType("chumpy.ch")}
    Ch.__module__, Ch.__qualname__ = "chumpy.ch", "Ch"
    mods["chumpy.ch"].Ch = Ch
    sys.modules.update(mods)
    try:
        obj = dict(raw, v_template=Ch(raw["v_template"]), shapedirs=Ch(raw["shapedirs"]), posedirs=Ch(raw["posedirs"]))
        for proto in (0, 2):
            with open(tmp_path / f"m{proto}.pkl", "wb") as f:
                pickle.dump(obj, f, protocol=proto)
    finally:
        for k in mods:
            del sys.modules[k]
    for proto in (0, 2):
        _check(load_smpl_model(str(tmp_path / f"m{proto}.pkl")), raw)


def test_refuses_foreign_globals(tmp_path):
    raw = synthetic()
    raw["evil"] = os.system                       # any global outside numpy / scipy.sparse / chumpy
    p = tmp_path / "evil.pkl"
    p.write_bytes(pickle.dumps(raw, protocol=2))
    with pytest.raises(pickle.UnpicklingError, match="posix.system|os.system"):
        load_smpl_model(str(p))
    buf = io.BytesIO()
    pickle.dump({"v_template": types.SimpleNamespace(a=1)}, buf)
    (tmp_path / "ns.pkl").write_bytes(buf.getvalue())
    with pytest.raises(pickle.UnpicklingError, match="SimpleNamespace"):
        load_smpl_model(str(tmp_path / "ns.pkl"))


def _bad(tmp_path, **change):
    raw = synthetic()
    for k, v in change.items():
        if v is None:
            del raw[k]
        else:
            raw[k] = v(raw[k]) if callable(v) else v
    np.savez(tmp_path / "m.npz", **raw)
    return str(tmp_path / "m.npz")


@pytest.mark.parametrize("key", ["v_template", "shapedirs", "posedirs", "J_regressor", "weights", "kintree_table"])
def test_missing_key(tmp_path, key):
    with pytest.raises(ValueError, match=key):
        load_smpl_model(_bad(tmp_path, **{key: None}))


@pytest.mark.parametrize("key,f", [("shapedirs", lambda a: a[:-1]), ("posedirs", lambda a: a[:, :, :200]), ("J_regressor", lambda a: a[:, :-1]),
                                   ("weights", lambda a: a[:, :23]), ("kintree_table", lambda a: a[:, :20]), ("shapedirs", lambda a: a[:, :, :9])])
def test_inconsistent_shapes(tmp_path, key, f):
    with pytest.raises(ValueError, match=key):
        load_smpl_model(_bad(tmp_path, **{key: f}))


def test_parent_after_child(tmp_path):
    def later(kt):
        kt = kt.copy()
        kt[0, 5] = 7
        return kt
    with pytest.raises(ValueError, match="kintree_table"):
        load_smpl_model(_bad(tmp_path, kintree_table=later))


@pytest.mark.parametrize("key", ["v_template", "shapedirs", "posedirs", "J_regressor", "weights"])
def test_non_finite(tmp_path, key):
    def nan(a):
        a = a.copy()
        a.flat[3] = np.nan
        return a
    with pytest.raises(ValueError, match=key):
        load_smpl_model(_bad(tmp_path, **{key: nan}))


def test_weight_rows_sum_to_one(tmp_path):
    def off(w):
        w = w.copy()
        w[4, 0] += 2e-6
        return w
    with pytest.raises(ValueError, match="weights"):
        load_smpl_model(_bad(tmp_path, weights=off))
    def tiny(w):
        w = w.copy()
        w[4, 0] += 5e-7
        return w
    load_smpl_model(_bad(tmp_path, weights=tiny))
