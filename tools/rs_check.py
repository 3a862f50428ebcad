"""Compare the resampler kernel families on the same seeded input (run once per B200A_RS value; outputs go to /tmp).
    B200A_RS=mma python tools/rs_check.py save;  B200A_RS=bf16 python tools/rs_check.py cmp
"""
import sys
import torch
sys.path.insert(0, ".")
import audio_b200.transforms as T

mode = sys.argv[1]
dev = "cuda:0"
cases = [(44100, 16000, 5, 220500), (44100, 16000, 3, 100001), (44100, 16000, 2, 441 * 32), (44100, 16000, 1, 300),
         (48000, 16000, 4, 96000), (16000, 8000, 4, 50000), (22050, 16000, 2, 66150)]
worst = 0.0
for i, (o, n, rows, length) in enumerate(cases):
    g = torch.Generator().manual_seed(100 + i)
    x = torch.randn(rows, length, generator=g).to(dev)
    try:
        y = T.Resample(o, n, resampling_method="sinc_interp_kaiser").to(dev)(x).cpu()
    except Exception as e:  # forced family does not apply to this ratio
        print(f"case {o}->{n} {rows}x{length}: {type(e).__name__}: {str(e)[:80]}")
        continue
    path = f"/tmp/rs_check_{i}.pt"
    if mode == "save":
        torch.save(y, path)
        print(f"case {o}->{n} {rows}x{length}: saved {tuple(y.shape)}")
    else:
        ref = torch.load(path)
        err = (y - ref).abs().max().item()
        rel = err / ref.abs().max().item()
        bad = int(((y - ref).abs() > 1e-4).sum())
        print(f"case {o}->{n} {rows}x{length}: max abs err {err:.3e} (rel to peak {rel:.3e}), >1e-4: {bad}, nan: {int(torch.isnan(y).sum())}")
        worst = max(worst, err)
if mode != "save":
    print("WORST", worst)
