"""Times the UNETR decoder's training step on the GPU: forward + backward per 1024x1024 image of the production plan
(interpolation upsampler) at B = 1 and 2, and the 3x3 weight-gradient kernel of the head block (128 -> 64 channels at 1024^2).
Medians over repeated windows of at least one second, timed with CUDA events.  Prints one JSON line per measurement."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from micro_sam_b200 import _lib, unetr  # noqa: E402


def timed(fn, windows=5, min_s=1.0):
    fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(windows):
        n, ms = 0, 0.0
        while ms < 1000 * min_s:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            torch.cuda.synchronize()
            ms += a.elapsed_time(b)
            n += 1
        out.append(ms / n)
    out.sort()
    return out[len(out) // 2], out


def main():
    dev = "cuda:0"
    d = unetr.TrainableUNETRDecoder(unetr.default_decoder_state(), device=dev)
    for B in (1, 2):
        z = torch.randn(B, 256, 64, 64, device=dev)
        dm = torch.randn(B, 3, 1024, 1024, device=dev)

        def step():
            d.forward(z)
            d.backward(dm)

        med, all_ = timed(step)
        print(json.dumps({"what": "decoder forward+backward", "B": B, "ms_per_image": med / B, "windows_ms": all_}))
    L = _lib.lib()
    B, H, W, C0, C1, cout = 1, 1024, 1024, 64, 64, 64
    dy = torch.randn(B, H, W, cout, device=dev).to(torch.bfloat16)
    x0 = torch.randn(B, H, W, C0, device=dev).to(torch.bfloat16)
    x1 = torch.randn(B, H, W, C1, device=dev).to(torch.bfloat16)
    ws = torch.empty(int(L.msam_ais_wgrad_workspace(cout, C0, C1, B, H, W, 3)), device=dev, dtype=torch.uint8)
    dw = torch.empty(cout, 9 * (C0 + C1), device=dev)

    def wg():
        _lib.check(L.msam_op_ais_wgrad(_lib.ptr(dy), cout, _lib.ptr(x0), C0, _lib.ptr(x1), C1, B, H, W, 3, _lib.ptr(ws), ws.numel(),
                                       _lib.ptr(dw), _lib.cur_stream()))

    med, all_ = timed(wg)
    flops = 2.0 * B * H * W * cout * 9 * (C0 + C1)
    print(json.dumps({"what": "wgrad 3x3 128->64 at 1024^2", "ms": med, "tflops": flops / med / 1e9, "windows_ms": all_}))


if __name__ == "__main__":
    main()
