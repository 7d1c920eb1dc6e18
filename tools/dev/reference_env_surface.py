"""What the reference's own env classes touch, and what of it this repo provides.

Static (ast) scan of the reference's `BaseJiminyEnv` / `WalkerJiminyEnv` / interfaces (SURVEY.md 8b: "pipelines and TOML
env configs load unchanged") for
  * the external modules they import (and whether this image has them),
  * the attributes they read on `jiminy_py.core` (alias `jiminy`) and `pinocchio` (alias `pin`),
  * the attributes they read on the engine / simulator / robot / state objects,
checked against jiminy_b200's single-env `Engine` facade, `RobotTable`, `StepperState` and `RobotState`.  Reads
the reference's sources (REF below); the report it prints is committed under profiles/.
"""
import ast
import importlib.util
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
REF = "/root/reference/python/gym_jiminy/common/gym_jiminy/common"
FILES = ["envs/generic.py", "envs/locomotion.py", "bases/interfaces.py"]


def scan(path):
    tree = ast.parse(open(path).read())
    imports, mod_attrs, obj_attrs = set(), {}, {}
    aliases = {}
    for node in ast.walk(tree):
        if isinstance(node, ast.Import):
            for a in node.names:
                imports.add(a.name.split(".")[0])
                aliases[a.asname or a.name.split(".")[0]] = a.name
        elif isinstance(node, ast.ImportFrom) and node.level == 0 and node.module:
            imports.add(node.module.split(".")[0])
            for a in node.names:
                mod_attrs.setdefault(node.module, set()).add(a.name)
        elif isinstance(node, ast.Attribute):
            v = node.value
            if isinstance(v, ast.Name) and v.id in ("jiminy", "pin"):
                mod_attrs.setdefault(aliases.get(v.id, v.id), set()).add(node.attr)
            # self.<obj>.<attr> and <obj>.<attr> for the objects of the step path
            name = None
            if isinstance(v, ast.Attribute) and isinstance(v.value, ast.Name) and v.value.id == "self":
                name = v.attr
            elif isinstance(v, ast.Name):
                name = v.id
            if name in ("simulator", "engine", "robot", "stepper_state", "robot_state", "_robot_state", "pinocchio_model",
                        "pinocchio_data"):
                obj_attrs.setdefault(name.lstrip("_"), set()).add(node.attr)
    return imports, mod_attrs, obj_attrs


def main():
    imports, mod_attrs, obj_attrs = set(), {}, {}
    for f in FILES:
        i, m, o = scan(os.path.join(REF, f))
        imports |= i
        for k, v in m.items():
            mod_attrs.setdefault(k, set()).update(v)
        for k, v in o.items():
            obj_attrs.setdefault(k, set()).update(v)
    std = set(sys.stdlib_module_names)
    print("== external modules imported by", ", ".join(FILES))
    for mod in sorted(imports - std):
        print(f"  {mod:12s} {'available' if importlib.util.find_spec(mod) else 'ABSENT in this image'}")
    print("\n== names used from jiminy_py.core / pinocchio / jiminy_py.*")
    for mod in sorted(mod_attrs):
        if mod.split(".")[0] in ("jiminy_py", "pinocchio"):
            print(f"  {mod}: {', '.join(sorted(mod_attrs[mod]))}")

    from jiminy_b200 import core, model as M, robots as R
    robot, _ = R.load_robot("anymal")
    eng = core.Engine.__new__(core.Engine)
    provided = {
        "engine": set(dir(core.Engine)) | {"robots", "robot_states", "stepper_state", "is_simulation_running", "log_data"},
        "robot": set(dir(robot)) | set(vars(robot)),
        "stepper_state": set(dir(core.StepperState(1, 1))),
        "robot_state": set(dir(core.RobotState(1, 1, 1, 2))),
    }
    print("\n== attributes read on the objects of the step path (+ provided / - missing on the jiminy_b200 facade)")
    for obj in ("engine", "robot", "stepper_state", "robot_state"):
        used = sorted(obj_attrs.get(obj, ()))
        have = [a for a in used if a in provided[obj]]
        miss = [a for a in used if a not in provided[obj]]
        print(f"  {obj}: + {', '.join(have) or '-'}")
        print(f"  {' ' * len(obj)}  - {', '.join(miss) or '(none)'}")
    for obj in ("simulator", "pinocchio_model", "pinocchio_data"):
        print(f"  {obj} (no counterpart object: `Simulator` / `pinocchio.Model` / `pinocchio.Data` themselves): "
              f"{', '.join(sorted(obj_attrs.get(obj, ()))) or '-'}")


if __name__ == "__main__":
    main()
