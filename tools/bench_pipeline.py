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

    python tools/bench_pipeline.py [--robot atlas|anymal] [--loop host|device] [--alternate R] [--n-env 4096]
                                   [--steps 10] [--warmup 3] [--duration-max 0.4]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# atlas.py:28-37, :77-78
MOTOR_POSITION_MARGIN, MOTOR_VELOCITY_SAFE_GAIN, MOTOR_VELOCITY_MAX, MOTOR_ACCELERATION_MAX = 0.02, 0.15, 4.0, 30.0
MAHONY_KP, MAHONY_KI = 0.75, 0.057
KEYS = [("states", "pd_controller"), ("measurements", "EncoderSensor"), ("features", "mahony_filter")]


def make_env(n_env: int, api_=None, robot: str = "atlas", loop: str = "host", duration_max: float = 20.0):
    from jiminy_b200 import envs, scenarios
    kw = dict(simulation_duration_max=duration_max, api_=api_)
    if robot == "anymal":
        from jiminy_b200.torch_envs import DeviceBatchedEnv
        return (DeviceBatchedEnv if loop == "device" else envs.BatchedJiminyEnv)(scenarios.make("anymal", n_env, seed=0), **kw)
    from jiminy_b200.torch_envs import DevicePDControlBatchedEnv
    sc = scenarios.make(robot, n_env, seed=0, contact_model="constraint", solver="euler_explicit", dt_max=0.005)
    return (DevicePDControlBatchedEnv if loop == "device" else envs.PDControlBatchedEnv)(
        sc, joint_position_margin=0.0, joint_velocity_limit=MOTOR_VELOCITY_MAX, joint_acceleration_limit=MOTOR_ACCELERATION_MAX,
        safety=dict(kp=1.0 / MOTOR_POSITION_MARGIN, kd=MOTOR_VELOCITY_SAFE_GAIN, soft_position_margin=0.0, soft_velocity_max=MOTOR_VELOCITY_MAX),
        order=1, mahony=(MAHONY_KP, MAHONY_KI), **kw)


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
        duration_max: float = 0.4) -> dict:
    import torch
    from jiminy_b200.envs import flatten_observation
    env = make_env(n_env, api_, robot, loop, duration_max)
    device = loop == "device"
    on_gpu = device and env.torch_device.type == "cuda"
    nm = env.robot.nmotors
    # the actions of the run, made before the clock starts (device loop: already on the device)
    if robot == "anymal":
        acts = [env.sc.sample_targets(k) for k in range(warmup + steps)]
    else:
        acts = [np.zeros((n_env, nm))] * (warmup + steps)      # `env.action` after reset: target velocities = 0
    if device:
        acts = [torch.as_tensor(a, device=env.torch_device) for a in acts]
    keys = KEYS if robot == "atlas" else [("states", "agent", "q"), ("states", "agent", "v")]
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
            "anymal PD standing (plain PD law), spring-damper contacts, runge_kutta_4 1 ms, per-step position targets")
    out = {"metric": "env_steps_per_sec", "unit": "env-steps/s", "value": n_env * steps / dt, "ms_per_step": 1e3 * dt / steps,
           "loop": loop, "robot": robot, "n_env": n_env, "steps": steps, "warmup": warmup,
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


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--n-env", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--loop", choices=("host", "device"), default="host")
    ap.add_argument("--robot", choices=("atlas", "anymal"), default="atlas")
    ap.add_argument("--alternate", type=int, default=0, metavar="R")
    ap.add_argument("--duration-max", type=float, default=0.4)
    a = ap.parse_args()
    kw = dict(n_env=a.n_env, steps=a.steps, warmup=a.warmup, robot=a.robot, duration_max=a.duration_max)
    res = alternate(a.alternate, **kw) if a.alternate > 0 else run(loop=a.loop, **kw)
    res.update(gpu_info())
    print(json.dumps(res))
