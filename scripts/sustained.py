import sys, os, subprocess, threading, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from raft_b200.distance import pairwise_distance
from raft_b200.common import DeviceResources
m = n = 100000; k = int(sys.argv[1]) if len(sys.argv) > 1 else 128; steps = int(sys.argv[2]) if len(sys.argv) > 2 else 60
h = DeviceResources()
g = torch.Generator(device="cuda").manual_seed(0)
x = torch.randn(m, k, device="cuda", generator=g) * 3; y = torch.randn(n, k, device="cuda", generator=g) * 3
out = torch.empty(m, n, device="cuda")
rows = []
proc = subprocess.Popen(["nvidia-smi", "--query-gpu=clocks.sm,power.draw,temperature.gpu,clocks_event_reasons.sw_power_cap,clocks_event_reasons.hw_slowdown,clocks_event_reasons.sw_thermal_slowdown", "--format=csv,noheader,nounits", "-lms", "20"], stdout=subprocess.PIPE, text=True)
threading.Thread(target=lambda: [rows.append((time.time(), l.strip())) for l in proc.stdout], daemon=True).start()
for _ in range(3): pairwise_distance(x, y, out=out, metric="sqeuclidean", handle=h)
torch.cuda.synchronize()
ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
t0 = time.time()
for a, b in ev:
    a.record(); pairwise_distance(x, y, out=out, metric="sqeuclidean", handle=h); b.record()
torch.cuda.synchronize(); t1 = time.time()
time.sleep(0.1); proc.terminate()
per = [a.elapsed_time(b) for a, b in ev]
print("per-step ms:", " ".join(f"{v:.2f}" for v in per))
print(f"first10 {sum(per[:10])/10:.3f}  last30 {sum(per[-30:])/30:.3f}  min {min(per):.3f}")
print("clock samples during run:", [r[1] for r in rows if t0 <= r[0] <= t1][::3])
