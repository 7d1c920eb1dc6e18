"""End-to-end timing of the reference's only published benchmark, restated over the batched engine.

`python/gym_jiminy/examples/pipeline_benchmark.py` steps `AtlasPDControlJiminyEnv` (MotorSafetyLimit + PDController +
PDAdapter(order=1) + MahonyFilter, atlas.py:239-295) behind FilterObservation / NormalizeObservation / FlattenObservation
with a constant action, 100 000 times: 27.4 s = 3.65 k env-steps/s on one CPU thread (BASELINE.md).  Here the same blocks
with the same arguments run for N lockstep envs: `PDControlBatchedEnv.step(action)` (host adapter, H2D of the target
accelerations, step kernel with controller / safety limits / observer inside, D2H of state, sensors, controller state and
filter state) followed by `flatten_observation` of the same three observation leaves.  Wall-clock, everything included.

The same loop runs host-bound (`--loop host`: numpy actions and observations, `envs.PDControlBatchedEnv`) or
device-resident (`--loop device`: torch tensors on the GPU, `torch_envs.DevicePDControlBatchedEnv`: the adapter, the
termination rule and the masked restart run on the device, no host synchronisation inside `step`).  `--robot anymal`
times the ANYmal headline configuration instead (PD standing, spring-damper contacts, RK4 1 ms) through
`envs.BatchedJiminyEnv` / `torch_envs.DeviceBatchedEnv` with per-step position targets.  Every env restarts inside the
timed window (`--duration-max`, default 0.4 s of simulated time).  `--alternate R` runs both loops R times in one process,
alternating, and reports each loop's spread.  The clock is the host's, around the step loop, ending in a device
synchronise.

`--disturbance R` turns the walker disturbance on (`std_ratio={"disturbance": R}`: impulses at 2 s intervals of simulated
time, none within the default `--duration-max`, and the profile evaluated at every dynamics evaluation, re-drawn at every
restart) and runs each loop with it off and on, alternating in one process, `max(--alternate, 1)` rounds.  On ANYmal the
forces ride the quadruped hot path (`env_step_kernel_ext`); Atlas runs the generic kernel either way.

`--sensors R` does the same for the walker sensor randomisation (`std_ratio={"sensors": R}`: per-env noise, bias, delay
and jitter of every sensor and fresh generator seeds, re-drawn at every restart); with both options both are on in the
"on" runs.

`--robot anymal_flexible` is the ANYmal configuration on the robot with a flexibility joint in every leg, and `--model R`
turns the walker model randomisation on the same way (`std_ratio={"model": R}`: per-env stiffness and damping of every
flexibility joint, re-drawn at every restart; r <= 2 on that robot).

`--model-bias S` sets the four body-bias standard deviations of the robot options (`massBodiesBiasStd`,
`centerOfMassPositionBodiesBiasStd`, `inertiaBodiesBiasStd`, `relativePositionBodiesBiasStd`) to S (`model_bias_std`:
per-env masses, centres of mass, inertias and joint placements, re-drawn at every restart) and runs each loop with them
off and on, alternating in one process, `max(--alternate, 1)` rounds; randomisation options given with it are on in both.

`--restart sample` times the device loop with its restarts from fresh draws of the initial-state distribution put on the
ground in the start kernel (`reset_states="sample"`) against the default restart bank, alternating in one process,
`max(--alternate, 1)` rounds; randomisation options given with it are on in both.

`--compositions` times the device loop without and with a representative composition spec (`jiminy_b200.compositions`:
roll-pitch, falling and mechanical-safety terminations, and an additive mixture of `SurviveReward` and
`MinimizeMechanicalPowerConsumption`), alternating in one process, `max(--alternate, 1)` rounds: the cost of the
contact-frame pass and the two composition launches per env-step.

`--stack NUM,SKIP` times the device loop without and with observation stacking (`jiminy_b200.observation_stack`,
num_stack NUM, skip_frames_ratio SKIP), alternating in one process, `max(--alternate, 1)` rounds.  The stacked leaves are
`t`, `measurements.ImuSensor` and 12 doubles of motor data, 19 doubles per frame: `measurements.EffortSensor` on the
plain-PD ANYmal and anymal_flexible envs, the PDController's action (`augment_observation=True`) on Atlas.

`--observers` times the device loop with the MahonyFilter on its default path (exact start, no twist removal, no rpy)
against the full observer set (`jiminy_b200.observers`: `MahonyFilter(exact_init=False, ignore_twist=True,
compute_rpy=True)` and `BodyObserver(twist_time_constant=0.3)`), alternating in one process, `max(--alternate, 1)` rounds:
the cost of the observers' refreshes inside the step kernel and of their observation leaves.  Atlas flattens the
filter's quaternion in both; the plain-PD ANYmal and anymal_flexible envs get the filter on their engine in both (their
observation does not include it).

    python tools/bench_pipeline.py [--robot atlas|anymal|anymal_flexible] [--loop host|device] [--alternate R]
                                   [--n-env 4096] [--steps 10] [--warmup 3] [--duration-max 0.4] [--disturbance R]
                                   [--sensors R] [--model R] [--model-bias S] [--restart bank|sample] [--compositions]
                                   [--stack NUM,SKIP] [--observers]
"""
import argparse
import json
import os
import sys
import time
from typing import Optional

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# atlas.py:28-37, :77-78
MOTOR_POSITION_MARGIN, MOTOR_VELOCITY_SAFE_GAIN, MOTOR_VELOCITY_MAX, MOTOR_ACCELERATION_MAX = 0.02, 0.15, 4.0, 30.0
MAHONY_KP, MAHONY_KI = 0.75, 0.057
KEYS = [("states", "pd_controller"), ("measurements", "EncoderSensor"), ("features", "mahony_filter")]


def make_env(n_env: int, api_=None, robot: str = "atlas", loop: str = "host", duration_max: float = 20.0,
             disturbance: float = 0.0, sensors: float = 0.0, model: float = 0.0, restart: str = "bank",
             model_bias: float = 0.0, compositions: bool = False, stack=None, observers=None):
    from jiminy_b200 import envs, scenarios
    from jiminy_b200.observers import BodyObserver, MahonyFilter
    from jiminy_b200.observation_stack import StackObservation
    from jiminy_b200.model_randomisation import BIAS_OPTIONS
    ratio = {k: r for k, r in (("disturbance", disturbance), ("sensors", sensors), ("model", model)) if r > 0}
    kw = dict(simulation_duration_max=duration_max, api_=api_, std_ratio=ratio or None,
              model_bias_std={k: model_bias for k in BIAS_OPTIONS} if model_bias > 0 else None)
    if restart == "sample":
        if loop != "device":
            raise ValueError("--restart sample is an option of the device loop")
        kw["reset_states"] = "sample"
    if compositions:
        kw.update(representative_compositions(0.04 if robot == "atlas" else 0.01))
    if stack is not None:
        motors = ("measurements", "EffortSensor") if robot != "atlas" else ("actions",)
        kw["stack"] = StackObservation(stack[0], [("t",), ("measurements", "ImuSensor"), motors], stack[1])
        if robot == "atlas":
            kw["augment_observation"] = True
    if robot in ("anymal", "anymal_flexible"):
        from jiminy_b200.torch_envs import DeviceBatchedEnv
        env = (DeviceBatchedEnv if loop == "device" else envs.BatchedJiminyEnv)(scenarios.make(robot, n_env, seed=0), **kw)
        if observers is not None:
            env.engine.set_mahony_filter_full(1.0, 0.1, exact_init=not observers, ignore_twist=observers, compute_rpy=observers)
            if observers:
                env.engine.set_body_observer(True, 0.3, True)
        return env
    if observers:
        kw["mahony"] = MahonyFilter(MAHONY_KP, MAHONY_KI, exact_init=False, ignore_twist=True, compute_rpy=True)
        kw["body_observer"] = BodyObserver(twist_time_constant=0.3)
    from jiminy_b200.torch_envs import DevicePDControlBatchedEnv
    sc = scenarios.make(robot, n_env, seed=0, contact_model="constraint", solver="euler_explicit", dt_max=0.005)
    return (DevicePDControlBatchedEnv if loop == "device" else envs.PDControlBatchedEnv)(
        sc, joint_position_margin=0.0, joint_velocity_limit=MOTOR_VELOCITY_MAX, joint_acceleration_limit=MOTOR_ACCELERATION_MAX,
        safety=dict(kp=1.0 / MOTOR_POSITION_MARGIN, kd=MOTOR_VELOCITY_SAFE_GAIN, soft_position_margin=0.0, soft_velocity_max=MOTOR_VELOCITY_MAX),
        order=1, **{"mahony": (MAHONY_KP, MAHONY_KI), **kw})


def representative_compositions(step_dt: float) -> dict:
    """Roll-pitch, falling and mechanical-safety terminations and an additive mixture of survive and power rewards."""
    from jiminy_b200 import compositions as CP
    reward = CP.AdditiveMixtureReward("reward_total", [CP.SurviveReward(), CP.MinimizeMechanicalPowerConsumption(
        cutoff=500.0, horizon=0.2)], weights=[0.5, 0.5])
    terms = [CP.BaseRollPitchTermination(low=[-0.4, -0.4], high=[0.4, 0.4], grace_period=step_dt),
             CP.FallingTermination(min_base_height=0.2), CP.MechanicalSafetyTermination(position_margin=0.02, velocity_max=8.0)]
    return dict(reward=reward, terminations=terms)


def gpu_info() -> dict:
    """Name and enforced power limit of GPU 0 (read-only queries)."""
    try:
        import pynvml as nv
        nv.nvmlInit()
        h = nv.nvmlDeviceGetHandleByIndex(0)
        name = nv.nvmlDeviceGetName(h)
        return {"gpu": name.decode() if isinstance(name, bytes) else name,
                "power_limit_w": nv.nvmlDeviceGetEnforcedPowerLimit(h) / 1000.0}
    except Exception:      # noqa: BLE001
        pass
    try:
        import subprocess
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
        return {"gpu": out[0], "power_limit_w": float(out[1])}
    except Exception:      # noqa: BLE001
        return {"gpu": None, "power_limit_w": None}


def run(n_env: int, steps: int, warmup: int, api_=None, robot: str = "atlas", loop: str = "host",
        duration_max: float = 0.4, disturbance: float = 0.0, sensors: float = 0.0, model: float = 0.0,
        restart: str = "bank", model_bias: float = 0.0, compositions: bool = False, stack=None, observers=None) -> dict:
    import torch
    from jiminy_b200.envs import flatten_observation
    env = make_env(n_env, api_, robot, loop, duration_max, disturbance, sensors, model, restart, model_bias, compositions, stack,
                   observers)
    device = loop == "device"
    on_gpu = device and env.torch_device.type == "cuda"
    nm = env.robot.nmotors
    # the actions of the run, made before the clock starts (device loop: already on the device)
    if robot != "atlas":
        acts = [env.sc.sample_targets(k) for k in range(warmup + steps)]
    else:
        acts = [np.zeros((n_env, nm))] * (warmup + steps)      # `env.action` after reset: target velocities = 0
    if device:
        acts = [torch.as_tensor(a, device=env.torch_device) for a in acts]
    keys = KEYS if robot == "atlas" else [("states", "agent", "q"), ("states", "agent", "v")]
    if robot == "atlas" and observers:
        keys = [("features", "mahony_filter", "quat") if k == ("features", "mahony_filter") else k for k in keys]
    low = {KEYS[0]: env.command_state_lower[:2]} if robot == "atlas" else None
    high = {KEYS[0]: env.command_state_upper[:2]} if robot == "atlas" else None

    def sync():
        if on_gpu:
            torch.cuda.synchronize()
        else:
            env.engine.synchronize()
    obs, _ = env.reset()
    flat = flatten_observation(obs, keys, low, high)
    n_done = 0
    for k in range(warmup):
        obs, *_ = env.step(acts[k])
        flat = flatten_observation(obs, keys, low, high)
    sync()
    dones = []
    t0 = time.perf_counter()
    for k in range(warmup, warmup + steps):
        obs, reward, terminated, truncated, info = env.step(acts[k])
        flat = flatten_observation(obs, keys, low, high)
        dones.append(terminated | truncated)
    sync()
    dt = time.perf_counter() - t0
    n_done = int(sum(int(d.sum()) for d in dones))
    status = np.asarray(env.engine.get_status())
    q = obs["states"]["agent"]["q"]
    q = q.cpu().numpy() if hasattr(q, "cpu") else q
    desc = (f"{robot} PD-control pipeline (MotorSafetyLimit + PDController + PDAdapter(order=1) + MahonyFilter), constraint "
            f"contacts, euler_explicit 5 ms" if robot == "atlas" else
            f"{robot} PD standing (plain PD law), spring-damper contacts, runge_kutta_4 1 ms, per-step position targets")
    out = {"metric": "env_steps_per_sec", "unit": "env-steps/s", "value": n_env * steps / dt, "ms_per_step": 1e3 * dt / steps,
           "loop": loop, "restart": restart, "stack": stack, "observers": observers, "robot": robot, "disturbance": disturbance, "sensors": sensors, "model": model, "model_bias": model_bias, "n_env": n_env, "steps": steps, "warmup": warmup,
           "timing": "host clock around env.step + flatten_observation, ending in a device synchronise",
           "config": {"workload": f"{desc}, {n_env} envs, step_dt {env.step_dt}, simulation_duration_max {duration_max}",
                      "env": type(env).__name__, "lane_plan": env.engine.describe(), "observation_width": int(flat.shape[1])},
           "envs_restarted": n_done, "envs_flagged": int(((status & ~8) != 0).sum()),
           "base_height_min": float(q[:, 2].min())}
    if robot == "atlas":
        out["published_reference"] = {"value": 100000 / 27.4, "unit": "env-steps/s", "source": "pipeline_benchmark.py:46, one CPU thread"}
    env.close()
    return out


def alternate(rounds: int, **kw) -> dict:
    """Both loops `rounds` times in this process, alternating (host first); each loop's env-steps/s with its spread."""
    runs = {"host": [], "device": []}
    for _ in range(rounds):
        for loop in ("host", "device"):
            runs[loop].append(run(loop=loop, **kw))
    out = {"metric": "env_steps_per_sec", "unit": "env-steps/s", "robot": kw.get("robot", "atlas"), "rounds": rounds}
    for loop, rs in runs.items():
        v = sorted(r["value"] for r in rs)
        out[loop] = {"median": float(np.median(v)), "min": v[0], "max": v[-1], "values": [r["value"] for r in rs],
                     "ms_per_step_median": float(np.median([r["ms_per_step"] for r in rs])),
                     "envs_restarted": [r["envs_restarted"] for r in rs], "envs_flagged": [r["envs_flagged"] for r in rs],
                     "config": rs[-1]["config"]}
    out["device_over_host_median"] = out["device"]["median"] / out["host"]["median"]
    return out


def alternate_randomisation(rounds: int, ratios: dict, loops, off: Optional[dict] = None, **kw) -> dict:
    """Each loop with the randomisation of `ratios` ({"disturbance": r}, {"sensors": r}, {"model": r},
    {"model_bias": s}, {"restart": "sample"}, {"compositions": True}, {"stack": (num, skip)} or {"observers": True}) off and
    on, `rounds` times in this process, alternating; env-steps/s and spread.  `off` keyword arguments are given to the off
    runs."""
    name = "_".join(ratios)
    runs = {(loop, on): [] for loop in loops for on in (False, True)}
    for _ in range(rounds):
        for loop in loops:
            for on in (False, True):
                runs[(loop, on)].append(run(loop=loop, **(ratios if on else off or {}), **kw))
    out = {"metric": "env_steps_per_sec", "unit": "env-steps/s", "robot": kw.get("robot", "atlas"), "rounds": rounds}
    for (loop, on), rs in runs.items():
        v = sorted(x["value"] for x in rs)
        out[f"{loop}_{name}_{'on' if on else 'off'}"] = {
            "median": float(np.median(v)), "min": v[0], "max": v[-1], "ms_per_step_median": float(np.median([x["ms_per_step"] for x in rs])),
            "envs_restarted": [x["envs_restarted"] for x in rs], "envs_flagged": [x["envs_flagged"] for x in rs],
            "config": rs[-1]["config"]}
    for loop in loops:
        out[f"{loop}_on_over_off_median"] = out[f"{loop}_{name}_on"]["median"] / out[f"{loop}_{name}_off"]["median"]
    return out


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--n-env", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--loop", choices=("host", "device"), default="host")
    ap.add_argument("--robot", choices=("atlas", "anymal", "anymal_flexible"), default="atlas")
    ap.add_argument("--alternate", type=int, default=0, metavar="R")
    ap.add_argument("--duration-max", type=float, default=0.4)
    ap.add_argument("--disturbance", type=float, default=0.0, metavar="R")
    ap.add_argument("--sensors", type=float, default=0.0, metavar="R")
    ap.add_argument("--model", type=float, default=0.0, metavar="R")
    ap.add_argument("--model-bias", type=float, default=0.0, metavar="S")
    ap.add_argument("--restart", choices=("bank", "sample"), default="bank")
    ap.add_argument("--compositions", action="store_true")
    ap.add_argument("--stack", type=str, default=None, metavar="NUM,SKIP")
    ap.add_argument("--observers", action="store_true")
    a = ap.parse_args()
    kw = dict(n_env=a.n_env, steps=a.steps, warmup=a.warmup, robot=a.robot, duration_max=a.duration_max)
    ratios = {k: r for k, r in (("disturbance", a.disturbance), ("sensors", a.sensors), ("model", a.model)) if r > 0}
    if a.stack is not None:
        num, skip = (int(x) for x in a.stack.split(","))
        res = alternate_randomisation(max(a.alternate, 1), {"stack": (num, skip)}, ("device",), **ratios, **kw)
        off, on = res["device_stack_off"], res["device_stack_on"]
        res["added_ms_per_env_step"] = on["ms_per_step_median"] - off["ms_per_step_median"]
    elif a.observers:
        res = alternate_randomisation(max(a.alternate, 1), {"observers": True}, ("device",), off={"observers": False},
                                      **ratios, **kw)
        off, on = res["device_observers_off"], res["device_observers_on"]
        res["added_ms_per_env_step"] = on["ms_per_step_median"] - off["ms_per_step_median"]
    elif a.compositions:
        res = alternate_randomisation(max(a.alternate, 1), {"compositions": True}, ("device",), **ratios, **kw)
        off, on = res["device_compositions_off"], res["device_compositions_on"]
        res["added_ms_per_env_step"] = on["ms_per_step_median"] - off["ms_per_step_median"]
    elif a.model_bias > 0:
        if a.restart == "sample":
            kw["restart"] = "sample"
        res = alternate_randomisation(max(a.alternate, 1), {"model_bias": a.model_bias},
                                      (a.loop,), **ratios, **kw)
    elif a.restart == "sample":
        res = alternate_randomisation(max(a.alternate, 1), {"restart": "sample"}, ("device",), **ratios, **kw)
    elif ratios:
        res = alternate_randomisation(max(a.alternate, 1), ratios, ("host", "device") if a.alternate > 0 else (a.loop,), **kw)
    else:
        res = alternate(a.alternate, **kw) if a.alternate > 0 else run(loop=a.loop, **kw)
    res.update(gpu_info())
    print(json.dumps(res))
