"""Multi-GPU observation exchange (`jb_peer_obs_*`, `jiminy_b200.parallel.ObservationExchange`) on a box with at
least two GPUs: one process per GPU, rendezvous on 127.0.0.1.  Run with `python -m pytest
tests/test_gpu_peer.py -m gpu`; skipped with fewer than two GPUs."""
import os
import subprocess
import sys
import textwrap

import pytest

from conftest import ROOT, has_cuda

pytestmark = pytest.mark.gpu


def _ngpu():
    if not has_cuda():
        return 0
    import torch
    return torch.cuda.device_count()


WORKER = textwrap.dedent("""
    import os, sys, time
    sys.path.insert(0, %r)
    import numpy as np, torch, torch.distributed as dist
    from jiminy_b200 import core, scenarios
    from jiminy_b200.parallel import ObservationExchange
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    case = os.environ["CASE"]
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", init_method="tcp://127.0.0.1:%%s" %% os.environ["PORT"], rank=rank, world_size=world,
                            device_id=torch.device("cuda", rank))
    n_env = 200                      # not a multiple of the envs per warp: the last warp is ragged
    sc = scenarios.make("anymal", n_env, seed=rank)
    eng = core.BatchedEngine(sc.robot, sc.options, n_env, device=rank)
    eng.set_pd_controller(sc.kp, sc.kd)
    eng.set_command(sc.target0)
    eng.start(sc.q0, sc.v0)
    xch = ObservationExchange(eng, rank, world, rank, prefer_peer=(case != "nccl"))
    assert xch.mode == ("nccl" if case == "nccl" else "peer"), (xch.mode, xch.note)
    rob = sc.robot
    iq = np.array([rob.idx_q[m.joint] for m in rob.motors])
    haa = [k for k, m in enumerate(rob.motors) if "HAA" in m.name]
    flagged = 0
    for k in range(6):
        act = sc.sample_targets(k)
        if case == "handoff":        # every third env leaves its joint bounds: fast body -> full body inside the launch
            for j in haa:
                act[::3, j] = rob.q_upper[iq[j]] + 0.3
        eng.set_command(act)
        dist.barrier()               # host-side skew between the two processes is not what is being timed
        t0 = time.perf_counter()
        eng.step(sc.step_dt)
        got = xch.gather()
        eng.synchronize()            # PeerTimeout if any rank's signal is missing
        dt = time.perf_counter() - t0
        assert dt < 1.0, f"step + exchange took {dt:.3f} s: a completion signal was late"
        got = got.clone()
        ref = xch.reference_gather()
        assert torch.equal(got, ref), f"rank {rank} step {k}: gathered observations differ from the all-gather"
        mine = torch.from_numpy(eng.get_sensors()).to(ref.device)
        assert torch.equal(ref[rank * n_env:(rank + 1) * n_env], mine)
        flagged = max(flagged, int((eng.get_status() & 8 != 0).sum()))
    if case == "handoff":
        assert flagged > 0, "no env reached its bounds: the hand-off case was not exercised"
    else:
        assert flagged == 0
    if case == "timeout":
        # rank 1 stops stepping: rank 0's wait must give up and the next synchronising call must say so
        dist.barrier()
        if rank == 0:
            eng.step(sc.step_dt)
            xch.gather()
            try:
                eng.synchronize()
            except core.PeerTimeout as e:
                print("TIMEOUT-RAISED", e, flush=True)
            else:
                raise AssertionError("missing peer signal went unnoticed")
        dist.barrier()
    dist.barrier()
    dist.destroy_process_group()
    print("OK", flush=True)
""") % ROOT


@pytest.mark.skipif(_ngpu() < 2, reason="needs two GPUs on one box")
@pytest.mark.parametrize("case", ["clean", "handoff", "nccl", "timeout"])
def test_peer_observation_exchange_two_gpus(tmp_path, case):
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    port = str(29500 + os.getpid() % 2000)
    procs = []
    for rank in range(2):
        env = dict(os.environ, RANK=str(rank), WORLD_SIZE="2", PORT=port, CASE=case,
                   JB_PEER_TIMEOUT_S="0.5" if case == "timeout" else "2.0")
        procs.append(subprocess.Popen([sys.executable, str(script)], env=env, stdout=subprocess.PIPE,
                                      stderr=subprocess.STDOUT, text=True))
    outs = []
    for p in procs:
        try:
            outs.append(p.communicate(timeout=240)[0])
        except subprocess.TimeoutExpired:
            p.kill()
            outs.append(p.communicate()[0] + "\n<killed: timeout>")
    for p, o in zip(procs, outs):
        assert p.returncode == 0 and "OK" in o, o
    if case == "timeout":
        assert "TIMEOUT-RAISED" in outs[0], outs[0]
