"""Multi-GPU host path: one process per GPU (torchrun), image rows sharded over ranks, ONE framebuffer gather.

The reference parallelises over independent row bands (raytracer.rs:254-262); here band b (band_rows rows) goes
to rank b mod world. The per-(pixel,sample) counter RNG makes every pixel independent of the partition, so the
gathered frame is bit-identical to the single-GPU frame. The only exchange step is the gather of the RGB8 (or
linear f32) shards to rank 0 — torch.distributed.gather (NCCL send/recv over NVLink; gloo on CPU in the tests).
"""
from __future__ import annotations

import os
from typing import Optional

import numpy as np
import torch
import torch.distributed as dist

from . import CUDA_STREAM_LEGACY, ResidentScene, Scene, make_options, shard_row_indices, shard_rows


def _torch_stream() -> int:
    return torch.cuda.current_stream().cuda_stream or CUDA_STREAM_LEGACY


def env_rank_world():
    return int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("LOCAL_RANK", "0"))


def init(backend: Optional[str] = None):
    rank, world, local = env_rank_world()
    if world > 1 and not dist.is_initialized():
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29511")
        if backend is None:
            backend = "nccl" if torch.cuda.is_available() else "gloo"
        if backend == "nccl":
            torch.cuda.set_device(local)
            dist.init_process_group(backend, device_id=torch.device("cuda", local))
        else:
            dist.init_process_group(backend)
    return rank, world, local


def padded_rows(height: int, world: int, band_rows: int) -> int:
    return max(shard_rows(height, r, world, band_rows) for r in range(world))


def gather_frame(shard: torch.Tensor, height: int, world: int, band_rows: int, rank: int, out: Optional[torch.Tensor] = None,
                 gather_buf: Optional[torch.Tensor] = None):
    """Gather the ranks' compact row shards ([rows_r, W, C]) to rank 0 and de-interleave them into [H, W, C].
    `shard` must already be padded to padded_rows() rows. Returns the frame on rank 0, None elsewhere."""
    if world == 1:
        return shard[:height]
    rows_max = shard.shape[0]
    if rank == 0:
        if gather_buf is None:
            gather_buf = torch.empty((world,) + tuple(shard.shape), dtype=shard.dtype, device=shard.device)
        dist.gather(shard, list(gather_buf.unbind(0)), dst=0)
        if out is None:
            out = torch.empty((height,) + tuple(shard.shape[1:]), dtype=shard.dtype, device=shard.device)
        if band_rows == 1:
            # row y lives at gather_buf[y % world, y // world]
            inter = gather_buf.transpose(0, 1).reshape((rows_max * world,) + tuple(shard.shape[1:]))
            out.copy_(inter[:height])
        else:
            for r in range(world):
                idx = torch.as_tensor(shard_row_indices(height, r, world, band_rows), device=shard.device)
                out[idx] = gather_buf[r, : idx.numel()]
        return out
    dist.gather(shard, None, dst=0)
    return None


class DistributedRenderer:
    """Scene resident on this rank's GPU; a frame = trace the rank's rows, gather RGB8 to rank 0.

    In a frame loop (`render_async`) the gather of frame k runs on a side stream while frame k+1 is already tracing:
    the shard buffers are double-buffered, so the only exchange step of the path never sits on the critical path."""

    def __init__(self, scene: Scene, band_rows: int = 1, variant: int = 0):
        self.rank, self.world, self.local = env_rank_world()
        self.scene = scene
        self.band_rows = band_rows
        self.h, self.w = scene.c.height, scene.c.width
        self.device = torch.device("cuda", self.local)
        torch.cuda.set_device(self.device)
        self.opts = make_options(device=self.local, rank=self.rank, world=self.world, band_rows=band_rows, variant=variant)
        self.resident = ResidentScene(scene, self.opts)
        self.rows = self.resident.rows
        self.rows_max = padded_rows(self.h, self.world, band_rows)
        # a ring of shard buffers deeper than the two frames in flight: frame k+2 does not have to wait for the gather of frame k
        # (which ends only when the SLOWEST rank has delivered frame k), so rank-to-rank jitter of up to two frames is absorbed
        self.n_shards = 4
        self.shards = [torch.zeros((self.rows_max, self.w, 3), dtype=torch.uint8, device=self.device) for _ in range(self.n_shards)]
        self.shard = self.shards[0]
        self.frame = torch.empty((self.h, self.w, 3), dtype=torch.uint8, device=self.device) if self.rank == 0 else None
        self.gbuf = torch.empty((self.world, self.rows_max, self.w, 3), dtype=torch.uint8, device=self.device) if (self.rank == 0 and self.world > 1) else None
        self.comm_stream = torch.cuda.Stream(device=self.device) if self.world > 1 else None
        self.frame_streams = [torch.cuda.Stream(device=self.device) for _ in range(2)]   # consecutive frames alternate streams
        self._traced = [torch.cuda.Event() for _ in range(self.n_shards)]     # shard k has been written by resolve
        self._gathered = [torch.cuda.Event() for _ in range(self.n_shards)]   # shard k has been consumed by the gather
        self._frame_no = 0

    def render(self) -> dict:
        """One frame on the current torch stream, blocking. Returns this rank's stats; rank 0's `frame` holds the image."""
        self.shard = self.shards[0]
        st = self.resident.render(self.shard.data_ptr(), 0, _torch_stream())
        if self.world > 1:
            gather_frame(self.shard, self.h, self.world, self.band_rows, self.rank, self.frame, self.gbuf)
        else:
            self.frame = self.shard[: self.h]
        return st

    def render_async(self):
        """Enqueue one frame without waiting. Frames alternate between two streams (and two shard buffers, and the
        library's two work-buffer sets), so frame k+1 starts tracing while frame k drains its last paths, resolves and
        is gathered on the side stream."""
        k = self._frame_no % self.n_shards
        fs = self.frame_streams[self._frame_no & 1]
        self._frame_no += 1
        cur = torch.cuda.current_stream()
        fs.wait_stream(cur)                                      # whatever the caller enqueued before this frame
        shard = self.shards[k]
        if self.world > 1 and self._frame_no > self.n_shards:
            fs.wait_event(self._gathered[k])                    # the gather n_shards frames ago has finished reading this shard
        self.resident.render_async(shard.data_ptr(), 0, fs.cuda_stream)
        self.shard = shard
        if self.world > 1:
            self._traced[k].record(fs)
            self.comm_stream.wait_event(self._traced[k])
            with torch.cuda.stream(self.comm_stream):
                gather_frame(shard, self.h, self.world, self.band_rows, self.rank, self.frame, self.gbuf)
                self._gathered[k].record(self.comm_stream)
        else:
            self.frame = shard[: self.h]

    def join(self):
        """Make the current stream wait for every frame enqueued so far (and its gather)."""
        cur = torch.cuda.current_stream()
        for fs in self.frame_streams:
            cur.wait_stream(fs)
        if self.comm_stream is not None:
            cur.wait_stream(self.comm_stream)

    def wait(self) -> dict:
        self.join()
        return self.resident.wait()

    def release(self):
        self.resident.release()
