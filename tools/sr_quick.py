"""tools/sr_quick.py -- one-process check of the SR head after a kernel change: the `const` case of tests/test_gpu_sr_native.py
(workspace activations + final image against the fp16 data-flow emulation, the fp32 convolutions and the reference golden) and the
SR head's ms/frame (CUDA events, 16 resident frames)."""
import os
import sys
import traceback

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import test_gpu_sr_native as T  # noqa: E402

try:
    T.test_native_sr_head_matches_emulation_and_fp32("const")
    print("PARITY OK")
except Exception:
    traceback.print_exc()
    print("PARITY FAILED")
net, _, _ = T._net()
net = net.cuda()
net.backend = "native"
rgb = torch.rand(16, 256 * 256, 3, device="cuda")
out = torch.empty(16, 3, 512, 512, device="cuda")
for _ in range(3):
    net.forward_native(rgb, noise_mode="const", clamp=True, out=out)
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(5):
    net.forward_native(rgb, noise_mode="const", clamp=True, out=out)
e1.record()
torch.cuda.synchronize()
print(f"SR head: {e0.elapsed_time(e1) / 5 / 16:.4f} ms/frame")
