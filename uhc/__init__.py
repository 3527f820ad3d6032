"""Drop-in `uhc` package: the Python surface scripts/train_uhc.py and scripts/eval_uhc.py of ZhengyiLuo/UHC import
(SURVEY.md section 8b), re-implemented on the batched engine (uhc_b200).  Only the hot path named by BASELINE.json lives here:
Config, flags, agent_dict / AgentCopycat, HumanoidEnv (single-env facade), reward registry, dataset loader; rendering entry
points are import-compatible shims."""
