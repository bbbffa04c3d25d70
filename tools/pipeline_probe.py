#!/usr/bin/env python3
"""Frame-loop timing of ONE GPU's share of an N-GPU run (shard 0 of `world`), pipelined over two streams like
rtb200/dist.py, without NCCL. usage: pipeline_probe.py [C2] [world] [frames]"""
import sys, os
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, 'rust-raytracer_b200'))
import torch
import rtb200 as R
from rtb200 import scenes
name = sys.argv[1] if len(sys.argv) > 1 else 'C2'
world = int(sys.argv[2]) if len(sys.argv) > 2 else 8
frames = int(sys.argv[3]) if len(sys.argv) > 3 else 40
sc = scenes.scene(name)
rs = R.ResidentScene(sc, R.make_options(rank=0, world=world))
rows = rs.rows
outs = [torch.zeros(rows * sc.c.width * 3, dtype=torch.uint8, device='cuda') for _ in range(2)]
streams = [torch.cuda.Stream() for _ in range(2)]
flush = torch.empty(160 << 20, dtype=torch.uint8, device='cuda')
def loop(n):
    cur = torch.cuda.current_stream()
    for k in range(n):
        flush.zero_()
        streams[k & 1].wait_stream(cur)
        rs.render_async(outs[k & 1].data_ptr(), 0, streams[k & 1].cuda_stream)
    for s in streams:
        cur.wait_stream(s)
loop(6); torch.cuda.synchronize(); rs.wait()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record(); loop(frames); e1.record(); torch.cuda.synchronize()
st = rs.wait()
ms = e0.elapsed_time(e1) / frames
print(f"{name} shard 0 of {world}: {ms:.3f} ms/frame pipelined, {st['rays'] / ms / 1e3:.0f} Mrays/s per GPU", flush=True)
