#!/usr/bin/env python
"""One benchmark step between cudaProfilerStart/Stop, for a profiler that honours them, e.g.
    ncu --profile-from-start off --metrics gpu__time_duration.sum --clock-control none --csv --log-file X python tools/one_step.py
(the launch list the roofline shares are checked against).  Reduced batch (same model, same chunk size,
one resident + one re-encoded chunk) so that the serialised capture stays within a minute or two."""
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import torch  # noqa: E402
import bench  # noqa: E402

batch = int(sys.argv[1]) if len(sys.argv) > 1 else 1536
mb = int(sys.argv[2]) if len(sys.argv) > 2 else 768
retain = int(sys.argv[3]) if len(sys.argv) > 3 else 1
dev = torch.device("cuda", 0)
torch.cuda.set_device(0)
run = bench.Runner(bench.WORKLOADS["cfg3"][0], "nce", batch, mb, 0.5, dev, 0, 1, retain=retain)
for _ in range(2):
    run.step()
torch.cuda.synchronize()
torch.cuda.profiler.start()
run.step()
torch.cuda.synchronize()
torch.cuda.profiler.stop()
print("plan", run.clip.last_step_plan)
