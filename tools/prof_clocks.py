#!/usr/bin/env python
"""Cycle accounting of the step kernel (development build, tools/build_prof.sh).

    python tools/prof_clocks.py [workload] [n_env] [steps]              # full body, contacts.model = constraint
    python tools/prof_clocks.py --hot-path [workload] [n_env] [steps]   # hot path, the scenario's spring-damper contacts

The default mode shows where a warp of the full body spends its cycles on the `constraint` contact model -- sweeps, bound
update, solver set-up, PGS sweep, refresh -- and how often its envs were in a solve together.  `--hot-path` gives the
budget of the hot-path body on the headline workload of bench.py: stepper calls (the RK4 stage calls), the controller
breakpoints (controller update, then the FSAL repair of the derivative), the sensor refresh and the rest of the step."""
import ctypes as C, os, sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from jiminy_b200 import scenarios, core
argv = sys.argv[1:]
hot = "--hot-path" in argv
argv = [a for a in argv if a != "--hot-path"]
name = argv[0] if len(argv) > 0 else "anymal"
n = int(argv[1]) if len(argv) > 1 else 4096
steps = int(argv[2]) if len(argv) > 2 else 3
NPROF = 24                                       # JB_PROF_N of jb_device.cuh
api = core.Api(C.CDLL(os.path.join(ROOT, "jiminy_b200", "libjiminy_b200_prof.so")))
api.dll.jb_debug_prof.argtypes = [C.c_void_p, C.POINTER(C.c_double)]
sc = scenarios.make(name, n) if hot else scenarios.make(name, n, contact_model="constraint")
eng = core.BatchedEngine(sc.robot, sc.options, n, api_=api)
if sc.kp is not None: eng.set_pd_controller(sc.kp, sc.kd)
eng.set_command(sc.target0); eng.start(sc.q0, sc.v0)
out = (C.c_double * NPROF)()
for k in range(2):
    eng.set_command(sc.sample_targets(k)); eng.step(sc.step_dt)
api.dll.jb_debug_prof(eng._h, out)          # clear
for k in range(steps):
    eng.set_command(sc.sample_targets(2 + k)); eng.step(sc.step_dt)
api.dll.jb_debug_prof(eng._h, out)
p = np.array(out[:]); warps = p[7] / steps
per = lambda i: p[i] / p[7]                    # per warp and launch
if hot:
    kern = per(6)
    rest = kern - (per(16) + per(17) + per(18) + per(20))
    share = lambda x: 100.0 * x / kern
    print(f"{name} x {n}, hot path ({sc.options['contacts']['model']} contacts): per warp and env-step "
          f"({int(warps)} warps, {steps} steps, {int((eng.get_status() != 0).sum())} envs with status bits)")
    print(f"  kernel                          {kern / 1e3:9.1f} k cycles")
    print(f"  stepper calls (RK4 stages)      {per(16) / 1e3:9.1f} k  {share(per(16)):5.1f} %   "
          f"{per(21):5.1f} calls, {per(16) / max(per(21), 1):7.0f} cycles each")
    print(f"  controller breakpoints          {(per(17) + per(18)) / 1e3:9.1f} k  {share(per(17) + per(18)):5.1f} %")
    print(f"    controller update             {per(17) / 1e3:9.1f} k  {share(per(17)):5.1f} %")
    print(f"    FSAL repair                   {per(18) / 1e3:9.1f} k  {share(per(18)):5.1f} %   "
          f"{per(19):5.1f} repairs, {per(18) / max(per(19), 1):7.0f} cycles each")
    print(f"  sensor refresh                  {per(20) / 1e3:9.1f} k  {share(per(20)):5.1f} %")
    print(f"  everything else                 {rest / 1e3:9.1f} k  {share(rest):5.1f} %")
    sys.exit(0)
print(f"{name} x {n}, contacts.model = constraint: per warp and env-step ({int(warps)} warps, {steps} steps)")
print(f"  kernel                {per(6) / 1e6:8.2f} M cycles")
print(f"  sweeps (rhs)          {per(0) / 1e6:8.2f} M   bound update {per(1) / 1e6:6.2f} M   votes + solver {per(2) / 1e6:6.2f} M")
print(f"  solver: set-up        {per(3) / 1e6:8.2f} M   sweep loop   {per(4) / 1e6:6.2f} M   refresh        {per(5) / 1e6:6.2f} M")
print(f"  rhs() calls           {per(8):8.1f}     lanes present per call {p[9] / max(p[8], 1):5.1f}")
print(f"  solves: whole warp    {per(10):8.1f}     partial warp {per(11):8.1f}     sweep iterations {per(12):9.1f}  ({per(12) / max(per(10) + per(11), 1):.1f} per solve)")
it = max(per(12), 1)
print(f"  cycles per sweep iteration {per(4) / it:8.0f}   per set-up {per(3) / max(per(10) + per(11), 1):8.0f}   per rhs sweeps {per(0) / max(per(8), 1):8.0f}")
print(f"  inside the sweep, per iteration: normal-force loop {p[13] / max(p[12], 1):7.0f}   friction loop {p[14] / max(p[12], 1):7.0f}   stopping criterion {p[15] / max(p[12], 1):7.0f}")
