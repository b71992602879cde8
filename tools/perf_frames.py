"""Frame preprocessing timing: the host path (Pillow, `vision_frames.process_frames`) against the GPU path
(`vision_frames.process_frames_cuda`), per frame, at 640x360, 1280x720 and 1920x1080 with T = 16 and 256 frames:
  host       Image.fromarray + process_frames on one CPU core (what a caller holding decord's uint8 arrays runs)
  gpu+upload process_frames_cuda from host uint8 frames: copy into pinned memory, upload, kernel (host clock around a
             device synchronise)
  gpu kernel process_frames_cuda from device-resident frames (CUDA events)
  pin copy / upload   the two halves of the upload alone: host copy into a pinned buffer, pinned -> device copy
Then frames -> codes for a 16-frame 720p clip both ways (synthetic VQGAN weights, default precision): whether the pixels
are identical, and how many codes differ between the two ways and between two encodes of the same pixels. Prints the
card, its power limit and max SM clock first.
Usage: python tools/perf_frames.py [--quick]"""
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from PIL import Image

from lwm_b200.vision_frames import process_frames, process_frames_cuda


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return "%s (nvidia-smi: %s)" % (torch.cuda.get_device_name(0), e)


def host_ms(fn, reps):
    """median wall time of fn() followed by a device synchronise"""
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return sorted(ts)[len(ts) // 2]


def event_ms(fn, reps):
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return sorted(ts)[len(ts) // 2]


def host_path(clip):
    return process_frames([Image.fromarray(f) for f in clip])


def main():
    quick = "--quick" in sys.argv
    print("card: %s" % card(), flush=True)
    rng = np.random.default_rng(0)
    for (w, h) in ((640, 360), (1280, 720), (1920, 1080)):
        for T in ((16,) if quick else (16, 256)):
            clip = rng.integers(0, 256, (T, h, w, 3), dtype=np.uint8)
            dev = torch.from_numpy(clip).cuda()
            pinned = torch.empty(clip.shape, dtype=torch.uint8, pin_memory=True)
            got = process_frames_cuda(clip)                                    # warm-up: tables, module, pinned pool
            process_frames_cuda(dev)
            torch.cuda.synchronize()
            t_host = host_ms(lambda: host_path(clip), 1 if T > 16 else 3)
            t_up = host_ms(lambda: process_frames_cuda(clip), 5)
            t_kern = event_ms(lambda: process_frames_cuda(dev), 20)
            t_pin = host_ms(lambda: pinned.copy_(torch.from_numpy(clip)), 5)
            t_dma = event_ms(lambda: pinned.to("cuda", non_blocking=True), 5)
            same = torch.equal(got[:4].cpu(), torch.from_numpy(host_path(clip[:4])))
            print("%4dx%-4d T=%3d  per frame: host %7.3f ms | gpu+upload %6.3f ms | gpu kernel %6.4f ms | "
                  "pin copy %6.3f ms, upload %6.3f ms (%.1f GB/s) | identical %s"
                  % (w, h, T, t_host / T, t_up / T, t_kern / T, t_pin / T, t_dma / T, clip.nbytes / t_dma / 1e6, same),
                  flush=True)
            del dev, pinned, got
            torch.cuda.empty_cache()

    from lwm_b200.vqgan import VQGAN, init_params
    tok = VQGAN(init_params(seed=0))
    clip = rng.integers(0, 256, (16, 720, 1280, 3), dtype=np.uint8)
    host = lambda: tok.encode(host_path(clip))[1]               # noqa: E731
    gpu = lambda: tok.encode(process_frames_cuda(clip))[1]      # noqa: E731
    same_pixels = torch.equal(process_frames_cuda(clip).cpu(), torch.from_numpy(host_path(clip)))
    idx_host, idx_gpu, idx_gpu2 = host(), gpu(), gpu()
    # the encoder's GroupNorm statistics are summed with float atomics, so even two encodes of the same pixels can
    # split a near-tie: count both
    print("16 x 1280x720: pixels identical %s; codes differing host vs GPU preprocessing %d, GPU vs GPU %d of %d"
          % (same_pixels, int((idx_host != idx_gpu).sum()), int((idx_gpu != idx_gpu2).sum()), idx_host.numel()),
          flush=True)
    t_host = host_ms(host, 3)
    t_gpu = host_ms(gpu, 3)
    dev = torch.from_numpy(clip).cuda()
    t_dev = event_ms(lambda: tok.encode(process_frames_cuda(dev)), 3)
    pixels = process_frames_cuda(dev)
    t_enc = event_ms(lambda: tok.encode(pixels), 3)
    print("frames -> codes, 16 x 1280x720 uint8 on the host: host preprocessing + encode %.1f ms | "
          "GPU preprocessing + encode %.1f ms | from device frames %.1f ms | encode alone %.1f ms"
          % (t_host, t_gpu, t_dev, t_enc), flush=True)


if __name__ == "__main__":
    main()
