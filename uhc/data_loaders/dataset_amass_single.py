"""DatasetAMASSSingle of the reference (uhc/data_loaders/dataset_amass_single.py:27-253): same pickle schema
{key: {pose_aa, pose_6d, trans, beta, gender, ...}}, same filtering (len >= t_min + 1), same sampling rules; in addition it
precomputes the expert tables of every clip once (uhc_b200.motion_lib) instead of once per episode, or, with
data_specs.expert_tables: device, hands the raw motion to the engine, which builds them on the GPU."""
import random

import joblib
import numpy as np

from uhc_b200 import motion_lib


def _gender_code(g):
    g = g.item() if isinstance(g, np.ndarray) else g
    if isinstance(g, bytes):
        g = g.decode("utf-8")
    return {"neutral": 0, "male": 1, "female": 2}[g]


class DatasetAMASSSingle:
    def __init__(self, data_specs, data_mode="train", model=None):
        np.random.seed(0)
        random.seed(0)
        self.data_root = data_specs["file_path"] if data_mode == "train" else data_specs["test_file_path"]
        self.data_specs = data_specs
        self.t_min, self.t_max = data_specs.get("t_min", 90), data_specs.get("t_max", -1)
        self.name = self.data_root.split("/")[-1]
        self.pickle_data = joblib.load(open(self.data_root, "rb"))
        self.data_mode = data_mode
        self.data, self.data_keys, self.sample_keys = {"pose_aa": {}, "trans": {}, "beta": {}, "gender": {}}, [], []
        for k, v in self.pickle_data.items():
            n = v["pose_aa"].shape[0]
            if n < self.t_min + 1:
                continue
            self.data["pose_aa"][k] = v["pose_aa"]
            self.data["trans"][k] = v["trans"] if v["trans"].shape[0] == n else v["qpos"][:, :3]
            beta = np.repeat(v["beta"][None], n, axis=0) if v["beta"].shape[0] != n else v["beta"]
            if beta.shape[1] != 16:
                beta = np.concatenate([beta, np.zeros((n, 16 - beta.shape[1]))], axis=1)
            self.data["beta"][k] = beta
            self.data["gender"][k] = np.repeat([_gender_code(v["gender"])], n, axis=0)
            self.data_keys.append(k)
            reps = n // self.t_max + 1 if self.t_max != -1 else 1
            self.sample_keys += [(k, [-1])] * reps
        self.seq_len = len(self.data_keys)
        self.curr_key = ""
        # expert tables of every clip, once (humanoid_im.py:182-215 does this per episode).  data_specs.expert_tables: "host" (default)
        # builds them here; "device" keeps only the raw motion (self.motions) and the engine builds the tables on the GPU (Engine.load_motions)
        self.expert_tables = data_specs.get("expert_tables", "host")
        assert self.expert_tables in ("host", "device"), "data_specs.expert_tables: host | device"
        if self.expert_tables == "device":
            self.motions = motion_lib.MotionSet([{"pose_aa": self.data["pose_aa"][k], "trans": self.data["trans"][k]} for k in self.data_keys])
        else:
            self.experts = [motion_lib.make_expert(self.data["pose_aa"][k], self.data["trans"][k], model) for k in self.data_keys]
        self.shapes = [np.concatenate([self.data["beta"][k][0], [self.data["gender"][k][0]]]) for k in self.data_keys]
        # opt-in height fix of raw motion against the floor (uhc_b200/motion_lib.py MotionSet.floor_audit / fix_height, on the GPU): it
        # needs the raw rows and an engine, so it runs in fix_floor once the engine exists
        self.fix_height = data_specs.get("fix_height", "off") or "off"
        self.drop_implausible = bool(data_specs.get("drop_implausible", False))
        assert self.fix_height in ("first_frame", "clip_min", "off"), "data_specs.fix_height: first_frame | clip_min | off"
        if (self.fix_height != "off" or self.drop_implausible) and self.expert_tables != "device":
            raise ValueError("data_specs.fix_height / data_specs.drop_implausible measure the raw motion on the GPU: they need "
                             "data_specs.expert_tables: device")
        self.floor_fixed = self.fix_height == "off" and not self.drop_implausible

    def fix_floor(self, engine, log=print):
        """data_specs.fix_height / drop_implausible, once: audits self.motions on the device, drops the clips the reference's rules drop
        (printed as process_amass_db.py prints them) and lowers the rest.  Returns True when the motion changed."""
        if self.floor_fixed:
            return False
        self.floor_fixed = True
        audit = self.motions.floor_audit(engine)
        drop = audit["implausible"] if self.drop_implausible else np.zeros(len(self.data_keys), bool)
        for c in np.flatnonzero(drop):
            k = self.data_keys[c]
            if audit["start_high"][c]:
                log(f"Starting too high: {k}")
            elif audit["airborne_run"][c] > self.motions.AIRBORNE_RUN:
                log(f"{k} too high sequence invalid for copycat: {audit['airborne_run'][c]}")
            else:
                log(f"{k} negative sequence invalid for copycat: {audit['deepest_toe'][c]}")
        for c in np.flatnonzero(audit["crawling"] & ~drop):
            log(f"Crawling: {self.data_keys[c]}")
        fixed = self.motions.fix_height(audit, self.fix_height)
        self.motions = fixed.drop(drop) if drop.any() else fixed
        gone = {k for k, d in zip(self.data_keys, drop) if d}
        self.data_keys = [k for k in self.data_keys if k not in gone]
        self.sample_keys = [s for s in self.sample_keys if s[0] not in gone]
        self.shapes = [s for s, d in zip(self.shapes, drop) if not d]
        adr = np.concatenate([[0], np.cumsum(self.motions.lens)])
        for c, k in enumerate(self.data_keys):          # the fixed translation, for get_sample_from_key
            self.data["trans"][k] = self.motions.rows[adr[c]:adr[c + 1], self.motions.pose_dim:self.motions.pose_dim + 3].copy()
        for k in gone:
            for d in self.data.values():
                d.pop(k)
        self.seq_len = len(self.data_keys)
        return True

    def get_len(self):
        return self.seq_len

    def get_sample_len_from_key(self, take_key):
        return self.data["pose_aa"][take_key].shape[0]

    def sample_seq(self, full_sample=False, freq_dict=None, sampling_temp=0.2, sampling_freq=0.5, precision_mode=False):
        self.curr_key = random.choice(self.sample_keys)[0]
        return self.get_sample_from_key(self.curr_key, full_sample=full_sample)

    def get_sample_from_key(self, take_key, full_sample=False, freq_dict=None, fr_start=-1, precision_mode=False, sampling_freq=0.75):
        self.curr_key = take_key
        n = self.data["pose_aa"][take_key].shape[0]
        if full_sample:
            fr_start, fr_end = 0, n
        else:
            if fr_start == -1:
                fr_start = np.random.randint(0, n - self.t_min)
            fr_end = fr_start + self.t_max if (fr_start + self.t_max < n and self.t_max != -1) else n
        self.fr_start, self.fr_end = fr_start, fr_end
        s = {k: self.data[k][take_key][fr_start:fr_end] for k in ("pose_aa", "trans", "beta", "gender")}
        s.update(seq_name=take_key, has_obj=False, num_obj=0, obj_pose=s["pose_aa"], clip_index=self.data_keys.index(take_key),
                 fr_start=fr_start)
        return s
