"""Multi-GPU layout of the batched step: envs are independent, so the batch is sharded by contiguous
env ranges, one process per GPU (`torch.distributed`, backend nccl; gloo in the CPU test-suite), with
no collective inside the physics.  The single exchange of the path is the end-of-step observation
concat (SURVEY.md 8e).  `ObservationExchange` is that exchange: by default the step kernel itself
stores every env's sensor row into the gathered buffer of every rank over NVLink / NVSwitch peer
memory (`jb_peer_obs_*`), falling back -- on all ranks together -- to one NCCL all-gather after the
step when the IPC mapping is unavailable.  `bench.py --gpus N` and the 2-GPU tests both go through it.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional, Tuple

import torch
import torch.distributed as dist


@dataclass(frozen=True)
class Shard:
    rank: int
    world: int
    n_total: int

    @property
    def bounds(self) -> Tuple[int, int]:
        """Contiguous env range [lo, hi) of this rank; sizes differ by at most one."""
        base, rem = divmod(self.n_total, self.world)
        lo = self.rank * base + min(self.rank, rem)
        return lo, lo + base + (1 if self.rank < rem else 0)

    @property
    def n_local(self) -> int:
        lo, hi = self.bounds
        return hi - lo

    def slice_actions(self, actions: torch.Tensor) -> torch.Tensor:
        """Every rank holds the replicated action tensor `[n_total, nmotors]`; it reads its own rows."""
        lo, hi = self.bounds
        return actions[lo:hi]


def gather_observations(local_obs: torch.Tensor, shard: Shard) -> torch.Tensor:
    """All-gather of `[n_local, width]` observation shards into `[n_total, width]`, global env order.
    Equal shards use one `all_gather_into_tensor` (a single NCCL all-gather over NVLink); ragged ones
    fall back to padded gathers."""
    if shard.world == 1:
        return local_obs
    width = local_obs.shape[1]
    base, rem = divmod(shard.n_total, shard.world)
    if rem == 0:
        out = torch.empty((shard.n_total, width), dtype=local_obs.dtype, device=local_obs.device)
        dist.all_gather_into_tensor(out, local_obs.contiguous())
        return out
    pad = torch.zeros((base + 1, width), dtype=local_obs.dtype, device=local_obs.device)
    pad[:local_obs.shape[0]] = local_obs
    parts = [torch.empty_like(pad) for _ in range(shard.world)]
    dist.all_gather(parts, pad)
    sizes = [Shard(r, shard.world, shard.n_total).n_local for r in range(shard.world)]
    return torch.cat([p[:n] for p, n in zip(parts, sizes)], dim=0)


class _DevArray:
    """Zero-copy torch view of a raw device pointer (CUDA array interface); fp64 unless `typestr` says otherwise."""

    def __init__(self, ptr: int, shape, typestr: str = "<f8"):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": typestr, "data": (int(ptr), False), "version": 3}


class ObservationExchange:
    """End-of-step observation concat of a sharded rollout (equal shards of `eng.n_env` envs per rank).

    mode "peer": the step kernel publishes the rows into every rank's buffer (no collective on the path);
    `gather()` only enqueues the wait for the other ranks' completion flags on the engine's stream.
    mode "nccl": `gather()` copies the sensor matrix and runs `all_gather_into_tensor`, ordered with the engine's
    stream on both sides.  Either way the returned `[world * n_env, width]` device tensor is valid once the engine's
    stream has reached that point (`eng.synchronize()` raises `PeerTimeout` if a rank never signalled).
    """

    def __init__(self, eng, rank: int, world: int, device: int, prefer_peer: bool = True):
        self.eng, self.rank, self.world, self.device = eng, rank, world, device
        self.mode, self.note = "none", "none (1 GPU)"
        self._in: Optional[torch.Tensor] = None
        self._out: Optional[torch.Tensor] = None
        if world == 1:
            return
        dev = torch.device("cuda", device)
        self.stream = torch.cuda.ExternalStream(eng.stream(), device=dev)
        self._in = torch.empty((eng.n_env, eng.width), dtype=torch.float64, device=dev)
        self._out = torch.empty((world * eng.n_env, eng.width), dtype=torch.float64, device=dev)
        self.mode, self.note = "nccl", "nccl all_gather_into_tensor after the step"
        if not prefer_peer:
            return
        ok = 1
        try:
            handle = eng.peer_obs_create(world, rank)
        except Exception as e:   # noqa: BLE001  (no peer access on this box: every rank falls back together)
            handle, ok, self.note = b"", 0, self.note + f" (peer_obs_create: {e})"
        handles = [None] * world
        dist.all_gather_object(handles, handle)
        if ok and all(len(h) == 64 for h in handles):
            try:
                eng.peer_obs_connect(handles)
            except Exception as e:   # noqa: BLE001
                ok, self.note = 0, self.note + f" (peer_obs_connect: {e})"
        else:
            ok = 0
        flag = torch.tensor([ok], device=dev)
        dist.all_reduce(flag, op=dist.ReduceOp.MIN)
        if int(flag.item()) == 1:
            self.mode = "peer"
            self.note = "in-kernel stores into peer memory (IPC-mapped gathered buffers), completion flags + wait kernel"
        else:
            if ok:
                eng.peer_obs_enable(False)   # this rank did connect: stop publishing so that all ranks run alike
            self.note += " (peer-memory exchange unavailable on this box)"

    def gather(self) -> Optional[torch.Tensor]:
        if self.mode == "peer":
            self.eng.peer_obs_wait()       # the rows were published by the step kernel itself
            return self.view()
        if self.mode == "nccl":
            self.eng.copy_sensors_to(self._in.data_ptr())
            ev = torch.cuda.Event()
            ev.record(self.stream)
            torch.cuda.current_stream().wait_event(ev)
            dist.all_gather_into_tensor(self._out, self._in)
            # the step kernel fills every SM's shared memory: a concurrent NCCL kernel would push its CTAs into a
            # second wave, so the next step is ordered after the gather
            done = torch.cuda.Event()
            done.record(torch.cuda.current_stream())
            self.stream.wait_event(done)
            return self._out
        return None

    def view(self) -> torch.Tensor:
        """Gathered observations of the last step, `[world * n_env, width]` (peer mode: the buffer the peers wrote)."""
        if self.mode == "peer":
            return torch.as_tensor(_DevArray(self.eng.peer_obs_view(), (self.world * self.eng.n_env, self.eng.width)),
                                   device=torch.device("cuda", self.device))
        return self._out

    def reference_gather(self) -> torch.Tensor:
        """Plain NCCL all-gather of the current sensor matrices (synchronous): what `view()` must equal."""
        self.eng.copy_sensors_to(self._in.data_ptr())
        self.eng.synchronize()
        dist.all_gather_into_tensor(self._out, self._in)
        torch.cuda.synchronize()
        return self._out
