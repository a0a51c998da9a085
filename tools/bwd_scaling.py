"""Backward-sweep time vs CTAs resident per SM: batch = (SM count)*k OCPs (one full wave of k CTAs/SM), k = 1..4.
Tells whether the kernel is latency-bound (time flat in k) or throughput-bound (time ~ k)."""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import numpy as np
import torch
from robotoc_b200 import ANYMAL, Layout, RiccatiRecursion
from helpers import trot_schedule
from synth import make_kkt
dims = ANYMAL; L = Layout(dims)
td, ev, ctrl = trot_schedule(40)
n_sm = torch.cuda.get_device_properties(0).multi_processor_count
base, dx0b = make_kkt(dims, L, ctrl, 8, 1)
for k in (1, 2, 3, 4, 8):
    batch = n_sm * k
    kkt = np.ascontiguousarray(np.tile(base, (batch // 8 + 1, 1, 1))[:batch])
    dx0 = np.ascontiguousarray(np.tile(dx0b, (batch // 8 + 1, 1))[:batch])
    rr = RiccatiRecursion(dims, len(ctrl), batch); rr.setTimeDiscretization(ctrl)
    rr.backwardRiccatiRecursion(kkt); rr.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ts = []
    for it in range(5):
        ev[0].record(); rr.backwardRiccatiRecursion(); ev[1].record(); torch.cuda.synchronize()
        ts.append(ev[0].elapsed_time(ev[1]))
    fw = []
    rr.forwardRiccatiRecursion(dx0); rr.synchronize()
    for it in range(5):
        ev[0].record(); rr.forwardRiccatiRecursion(); ev[1].record(); torch.cuda.synchronize()
        fw.append(ev[0].elapsed_time(ev[1]))
    print(f"k={k} batch={batch}: backward {min(ts):.3f} ms  ({min(ts)*1e3/len(ctrl):.2f} us/stage, {batch/min(ts):.0f} OCP/ms)   forward {min(fw):.3f} ms", flush=True)
    rr.close()
