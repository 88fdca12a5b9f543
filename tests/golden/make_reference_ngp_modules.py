"""Records what the reference's models/networks/ngp.py asks of tiny-cuda-nn: for every `self.<name> = tcnn.<Class>(...)`
in NeRFNGPNet.__init__ the attribute name, the class and its (literal) keyword arguments, and the names of the buffers
it registers -> tests/golden/reference_ngp_modules.json.  Needs /root/reference; only those constructor arguments are
stored, no source."""
import ast
import json
import os

SRC = "/root/reference/instant_avatar/models/networks/ngp.py"
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference_ngp_modules.json")

tree = ast.parse(open(SRC).read())
cls = next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == "NeRFNGPNet")
init = next(n for n in cls.body if isinstance(n, ast.FunctionDef) and n.name == "__init__")
modules, buffers = [], []
for node in ast.walk(init):
    if (isinstance(node, ast.Assign) and isinstance(node.value, ast.Call) and isinstance(node.value.func, ast.Attribute)
            and isinstance(node.value.func.value, ast.Name) and node.value.func.value.id == "tcnn"):
        modules.append({"attr": node.targets[0].attr, "class": node.value.func.attr,
                        "kwargs": {k.arg: ast.literal_eval(k.value) for k in node.value.keywords}})
    if isinstance(node, ast.Call) and isinstance(node.func, ast.Attribute) and node.func.attr == "register_buffer":
        buffers.append(ast.literal_eval(node.args[0]))
with open(OUT, "w") as fh:
    json.dump({"class": "NeRFNGPNet", "modules": modules, "buffers": buffers}, fh, indent=1)
    fh.write("\n")
print(OUT)
