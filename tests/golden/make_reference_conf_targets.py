"""Records the `_target_` strings of the reference's YAML configs (confs/{renderer,deformer,network}/*.yaml and the
top-level model configs) into tests/golden/reference_conf_targets.json, so that the import-surface test can check the
mirror against them without the reference tree.  Needs /root/reference; only the target strings are stored."""
import json
import os
import re

REF = "/root/reference"
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference_conf_targets.json")


def targets(path):
    return [m.group(1) for m in re.finditer(r"_target_:\s*(\S+)", open(path).read())]


out = {"by_subdir": [], "top_level": {}}
for sub in ("renderer", "deformer", "network"):
    d = os.path.join(REF, "confs", sub)
    for f in sorted(os.listdir(d)):
        out["by_subdir"] += [[f"confs/{sub}/{f}", t] for t in targets(os.path.join(d, f))]
for f in ("SNARF_NGP.yaml", "SNARF_NGP_refine.yaml", "SNARF_NGP_fitting.yaml", "demo.yaml"):
    out["top_level"][f"confs/{f}"] = targets(os.path.join(REF, "confs", f))
with open(OUT, "w") as fh:
    json.dump(out, fh, indent=1)
    fh.write("\n")
print(OUT)
