# coding=utf-8
"""One forward of a bench workload inside a cudaProfilerStart/Stop range (for ncu
--profile-from-start off).  Usage: python tools/profile_step.py --workload c4 --global-batch 128"""
import argparse, os, sys
import numpy as np
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench
from multiverse_b200 import synthetic
from multiverse_b200.engine import ConvRNNEngine

ap = argparse.ArgumentParser()
ap.add_argument("--workload", default="c4")
ap.add_argument("--global-batch", type=int, default=128)
a = ap.parse_args()
wl = bench.WORKLOADS[a.workload]
cfg = synthetic.make_config(batch_size=a.global_batch, **wl["cfg"])
dev = torch.device("cuda:0")
w = synthetic.make_weights(cfg)
f = synthetic.make_feeds(cfg, a.global_batch)
g = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)
feeds = dict(scene_feat=g(f["scene_feat"]), obs_scene=g(f["obs_scene"]),
             grid_obs_labels=[g(x) for x in f["grid_obs_labels"]], grid_obs_regress=[g(x) for x in f["grid_obs_regress"]])
eng = ConvRNNEngine(cfg, {k: torch.from_numpy(v) for k, v in w.items()}, dev)
for _ in range(2):
  eng.forward(feeds)
torch.cuda.synchronize()
torch.cuda.profiler.start()
eng.forward(feeds)
torch.cuda.synchronize()
torch.cuda.profiler.stop()
print("done")
