"""Records the `_target_` strings and arguments of the reference's dataset and sampler configs
(confs/dataset/*/*.yaml, confs/sampler/*.yaml) into tests/golden/reference_data_conf_targets.json, so that the import-surface
test can check them without the reference tree.  Needs /root/reference and PyYAML; only targets and scalar arguments are
stored."""
import json
import os

import yaml

REF = "/root/reference"
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference_data_conf_targets.json")

out = {"dataset": [], "sampler": []}
for sub in ("dataset", "sampler"):
    d = os.path.join(REF, "confs", sub)
    for dp, _, fs in sorted(os.walk(d)):
        for f in sorted(fs):
            cfg = yaml.safe_load(open(os.path.join(dp, f)))
            rel = os.path.relpath(os.path.join(dp, f), REF)
            args = {k: v for k, v in cfg.items() if k != "_target_" and not isinstance(v, dict)} if sub == "sampler" else {}
            out[sub].append([rel, cfg["_target_"], args])
with open(OUT, "w") as fh:
    json.dump(out, fh, indent=1)
    fh.write("\n")
print(OUT)
