"""GPU: the drop-in's evaluation sharded over W ranks (AgentCopycat at WORLD_SIZE > 1) against one rank, exactly.

W processes on the one GPU form a gloo group and each builds the same AgentCopycat on the same synthetic clips, with the weights of one
checkpoint the test writes.  Every env's roll-out is independent of the other envs and of its slot, so each clip gives the same bits on
whichever rank and in whichever call it runs: eval_policy's results, dumps and curriculum, eval_checkpoints, export_motion and the
rendered videos must all equal those of world 1, computed here in the test's own process, with == and not a tolerance."""
import datetime
import itertools
import os
import pickle
import socket
import types

import joblib
import numpy as np
import pytest

from tests.helpers import write_synthetic_pkl

pytestmark = pytest.mark.gpu

NUM_ENVS = 4                       # below a rank's share of the 11 training clips, so a rank makes several calls
SHORT = (12, 25, 7, 60, 33)        # frame counts of the first training clips: mixed lengths beside the 40-90 frames of the others
COMBOS = list(itertools.product((True, False), (True, False)))      # (fail_safe, eval_on_device)
PIECE = 150_000                    # max_bytes of the trajectory pieces: several pieces per rank
SIZE = (160, 90)


def _data(root):
    os.makedirs(root, exist_ok=True)
    train, test = os.path.join(root, "clips.pkl"), os.path.join(root, "test_clips.pkl")
    write_synthetic_pkl(train, nclips=11, seed=0)
    d = joblib.load(train)
    for key, T in zip(sorted(d), SHORT):
        for f in ("pose_aa", "pose_6d", "trans"):
            d[key][f] = d[key][f][:T]
    joblib.dump(d, train)
    write_synthetic_pkl(test, nclips=5, seed=1)
    tiny = os.path.join(root, "tiny_clips.pkl")      # fewer clips than ranks at W = 3: a rank with an empty shard
    write_synthetic_pkl(tiny, nclips=2, seed=2)
    return train, test, tiny


def _cfg(data, cur_dev):
    import yaml
    from uhc.utils.config_utils.copycat_config import Config
    base = yaml.safe_load(open(os.path.join(os.path.dirname(__file__), "..", "config", "uhc_b200_default.yml")))
    base.update(policy_hsize=[128, 64], value_hsize=[128, 64], min_batch_size=1024, num_optim_epoch=2, num_envs=NUM_ENVS, save_n_epochs=2, num_epoch=1)
    base["data_specs"].update(file_path=data[0], test_file_path=data[1], t_max=40, t_min=1, expert_tables="host")
    base.update(body_diff_thresh_test=0.2, eval_dump_motion=True, curriculum_on_device=cur_dev)    # failures within a few dozen frames
    cfg = Config(cfg_id="eval_shard", create_dirs=True, cfg_dict=base)
    cfg.update(types.SimpleNamespace(cfg="eval_shard", render=False, test=False, num_threads=4, gpu_index=0, epoch=0, show_noise=False,
                                     resume=None, no_log=True, debug=False, full_eval=False))
    return cfg


def _run(workdir, data, shared, cur_dev, video_dir):
    """the same sequence of evaluations at any world: returns everything the test compares"""
    import torch
    import uhc.agents.agent_copycat as ac
    os.makedirs(workdir, exist_ok=True)
    os.chdir(workdir)
    cfg = _cfg(data, cur_dev)
    agent = ac.AgentCopycat(cfg, torch.float64, torch.device("cuda", 0), training=True, checkpoint_epoch=0)
    with open(os.path.join(shared, "models", "iter_0001.p"), "rb") as f:
        agent.agent.load_state_dicts(pickle.load(f))
    names = [ld.name for ld in agent.test_data_loaders]
    seen = {"eval": [], "evaluate_policies": [], "render_motion": []}       # the clips this rank evaluated, per call, in call order
    eval_loader = agent._eval_loader

    def recording_eval_loader(loader, dump):
        res, pending = eval_loader(loader, dump)
        seen["eval"].append((loader.name, sorted(res)))
        return res, pending
    agent._eval_loader = recording_eval_loader
    for name, arg in (("evaluate_policies", 1), ("render_motion", 0)):
        def recording(*a, _fn=getattr(agent.agent, name), _name=name, _arg=arg, **kw):
            seen[_name].append(sorted(int(c) for c in np.atleast_1d(a[_arg])))
            return _fn(*a, **kw)
        setattr(agent.agent, name, recording)
    rec = {"eval": [], "seen": seen}
    for j, (fs, od) in enumerate(COMBOS):
        cfg.fail_safe = fs
        cfg.cfg_dict["eval_on_device"] = od
        res = agent.eval_policy(epoch=10 + j, dump=True, max_bytes=PIECE)
        pk = {n: joblib.load(p) for n in names if os.path.exists(p := os.path.join(cfg.output_dir, f"{10 + j}_{n}_coverage_full.pkl"))}
        cur = agent.agent.curriculum_get() if cur_dev else {k: [list(r) for r in v] for k, v in agent.freq_dict.items()}
        rec["eval"].append((res, pk, cur))
    cfg.fail_safe = True
    cfg.model_dir = os.path.join(shared, "models")
    rec["checkpoints"] = agent.eval_checkpoints([1, 2], dump=True)
    rec["checkpoint_pkl"] = {(e, n): joblib.load(p) for e in (1, 2) for n in names
                             if os.path.exists(p := os.path.join(cfg.output_dir, f"{e}_{n}_coverage_full.pkl"))}
    rec["export"] = agent.export_motion(epoch=7, dump=True, max_bytes=PIECE)
    rec["export_pkl"] = {n: joblib.load(p) for n in names if os.path.exists(p := os.path.join(cfg.output_dir, f"7_{n}_motion.pkl"))}
    rec["render"] = agent.render_motion(epoch=8, loaders=agent.test_data_loaders[1:], out_dir=video_dir, size=SIZE, video="mjpeg")
    from uhc.data_loaders.dataset_amass_single import DatasetAMASSSingle
    tiny = DatasetAMASSSingle(dict(cfg.data_specs, test_file_path=data[2]), data_mode="test", model=agent.model_tables)
    tiny.fix_floor(agent.agent.engine, agent.logger.info)
    rec["tiny_export"] = agent.export_motion(epoch=9, loaders=[tiny], dump=True, max_bytes=PIECE)[tiny.name]
    rec["tiny_export_pkl"] = joblib.load(p) if os.path.exists(p := os.path.join(cfg.output_dir, f"9_{tiny.name}_motion.pkl")) else None
    rec["tiny_render"] = agent.render_motion(epoch=9, loaders=[tiny], out_dir=video_dir, size=SIZE, video="mjpeg")[tiny.name]
    rec["keys"] = {ld.name: list(ld.data_keys) for ld in agent.test_data_loaders}
    rec["tiny_keys"] = list(tiny.data_keys)
    agent.agent.engine.close()
    return rec


def _child(rank, world, port, workdir, data, shared, cur_dev):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=datetime.timedelta(seconds=600))
    try:
        rec = _run(workdir, data, shared, cur_dev, os.path.join(shared, "videos_sharded"))
        joblib.dump(rec, os.path.join(shared, f"rank{rank}.pkl"))
    finally:
        dist.destroy_process_group()


def _same(a, b, path="."):
    """exact equality of nested results: same keys in the same order, same dtypes and shapes, equal bits (NaN equal to NaN)"""
    if isinstance(a, dict):
        assert isinstance(b, dict) and list(a) == list(b), (path, list(a), list(b) if isinstance(b, dict) else type(b))
        for k in a:
            _same(a[k], b[k], f"{path}/{k}")
    elif isinstance(a, (list, tuple)):
        assert type(a) is type(b) and len(a) == len(b), path
        for i, (x, y) in enumerate(zip(a, b)):
            _same(x, y, f"{path}[{i}]")
    elif isinstance(a, np.ndarray):
        assert isinstance(b, np.ndarray) and a.dtype == b.dtype and a.shape == b.shape, path
        assert np.array_equal(a, b, equal_nan=a.dtype.kind in "fc"), path
    elif isinstance(a, float):
        assert isinstance(b, float) and (a == b or (a != a and b != b)), (path, a, b)
    else:
        assert a == b, (path, a, b)


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close()
    return p


@pytest.mark.parametrize("world,cur_dev", [(2, False), (3, True)])
def test_sharded_evaluation_equals_one_rank(tmp_path, monkeypatch, world, cur_dev):
    import torch
    import torch.multiprocessing as mp
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    monkeypatch.delenv("RANK", raising=False)
    data = _data(str(tmp_path / "data"))
    shared = str(tmp_path / "shared")
    os.makedirs(os.path.join(shared, "models"))
    monkeypatch.chdir(tmp_path)

    # the one checkpoint every process evaluates, and a second one for eval_checkpoints
    import uhc.agents.agent_copycat as ac
    os.makedirs(tmp_path / "init")
    monkeypatch.chdir(tmp_path / "init")
    a0 = ac.AgentCopycat(_cfg(data, cur_dev), torch.float64, torch.device("cuda", 0), training=True, checkpoint_epoch=0)
    cp = a0.agent.state_dicts()
    with open(os.path.join(shared, "models", "iter_0001.p"), "wb") as f:
        pickle.dump(cp, f)
    cp["policy_dict"] = {k: (v * 1.05 if k != "action_log_std" else v) for k, v in cp["policy_dict"].items()}
    with open(os.path.join(shared, "models", "iter_0002.p"), "wb") as f:
        pickle.dump(cp, f)
    a0.agent.engine.close()
    del a0

    one = _run(str(tmp_path / "w1"), data, shared, cur_dev, os.path.join(shared, "videos_w1"))

    ctx = mp.get_context("spawn")
    port = _free_port()
    ps = [ctx.Process(target=_child, args=(r, world, port, str(tmp_path / f"rank{r}"), data, shared, cur_dev)) for r in range(world)]
    [p.start() for p in ps]
    try:
        for p in ps:
            p.join(1200)
    finally:
        for p in ps:
            if p.is_alive():
                p.terminate()
                p.join(30)
    assert [p.exitcode for p in ps] == [0] * world, [p.exitcode for p in ps]
    recs = [joblib.load(os.path.join(shared, f"rank{r}.pkl")) for r in range(world)]

    names = list(one["keys"])
    for r, rec in enumerate(recs):
        for j, ((res1, pk1, cur1), (res, pk, cur)) in enumerate(zip(one["eval"], rec["eval"])):
            _same(res1, res, f"rank {r} eval {COMBOS[j]} res_dicts")
            _same(cur1, cur, f"rank {r} eval {COMBOS[j]} curriculum")
            if r == 0:
                assert list(pk) == names
                _same(pk1, pk, f"eval {COMBOS[j]} coverage pickle")
            else:
                assert pk == {}, f"rank {r} wrote a coverage pickle"
        _same(one["checkpoints"], rec["checkpoints"], f"rank {r} eval_checkpoints")
        if r == 0:
            _same(one["checkpoint_pkl"], rec["checkpoint_pkl"], "eval_checkpoints pickles")
            _same(one["export"], rec["export"], "export_motion")
            _same(one["export_pkl"], rec["export_pkl"], "export_motion pickles")
        else:
            assert rec["checkpoint_pkl"] == {} and rec["export_pkl"] == {}
            for n in names:                                     # every other rank returns its own clips, in clip order
                own = list(rec["export"][n])
                assert own and own == [k for k in one["keys"][n] if k in own]
                _same({k: one["export"][n][k] for k in own}, rec["export"][n], f"rank {r} export_motion")
        assert {n: {k: os.path.basename(f) for k, f in p.items()} for n, p in rec["render"].items()} == \
            {n: {k: os.path.basename(f) for k, f in p.items()} for n, p in one["render"].items()}
    # the other ranks' own clips of the export: each clip at most once, and none of rank 0's
    for n in names:
        got = [k for rec in recs[1:] for k in rec["export"][n]]
        assert len(got) == len(set(got)) and set(got) < set(one["keys"][n])

    d1, dw = os.path.join(shared, "videos_w1"), os.path.join(shared, "videos_sharded")
    files = sorted(os.listdir(d1))
    assert files and files == sorted(os.listdir(dw))
    for f in files:
        with open(os.path.join(d1, f), "rb") as x, open(os.path.join(dw, f), "rb") as y:
            assert x.read() == y.read(), f

    # the work was split: in every call, the clips the ranks evaluated are a partition of the clips one rank evaluates, over >= 2 ranks
    for kind in ("eval", "evaluate_policies", "render_motion"):
        assert all(len(rec["seen"][kind]) == len(one["seen"][kind]) for rec in recs), kind
        for i, full in enumerate(one["seen"][kind]):
            per = [rec["seen"][kind][i] for rec in recs]
            if kind == "eval":
                assert all(name == full[0] for name, _ in per), (kind, i)
                full, per = full[1], [keys for _, keys in per]
            got = [c for p in per for c in p]
            assert sorted(got) == sorted(full) and len(got) == len(set(got)), (kind, i)
            assert sum(1 for p in per if p) >= 2, (kind, i, per)

    # a table with fewer clips than ranks (at W = 3 the last rank's shard is empty): export and render still equal world 1
    assert (world > len(one["tiny_keys"])) == (world == 3)
    _same(one["tiny_export"], recs[0]["tiny_export"], "export_motion, tiny table")
    _same(one["tiny_export_pkl"], recs[0]["tiny_export_pkl"], "export_motion pickle, tiny table")
    assert all(rec["tiny_export_pkl"] is None for rec in recs[1:])
    got = [k for rec in recs[1:] for k in rec["tiny_export"]]
    assert len(got) == len(set(got)) and set(got) <= set(one["tiny_keys"])
    if world == 3:
        assert recs[2]["tiny_export"] == {} and recs[2]["seen"]["render_motion"][-1] == []
    for rec in recs:
        assert {k: os.path.basename(f) for k, f in rec["tiny_render"].items()} == {k: os.path.basename(f) for k, f in one["tiny_render"].items()}
