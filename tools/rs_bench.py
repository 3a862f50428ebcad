import torch, sys
sys.path.insert(0, ".")
import audio_b200.transforms as T
dev="cuda:0"
r = T.Resample(44100, 16000, resampling_method="sinc_interp_kaiser").to(dev)
x = torch.randn(1024, 220500, device=dev)
for _ in range(3): y = r(x)
torch.cuda.synchronize()
e0,e1=torch.cuda.Event(enable_timing=True),torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(10): y = r(x)
e1.record(); torch.cuda.synchronize()
ms=e0.elapsed_time(e1)/10
print("resample C3 ms", ms, "GB/s", 1230.85e6/ms/1e6, "frac of the H100 SXM data-sheet 3350 GB/s", 1230.85e6/ms/1e6/3350.0)
