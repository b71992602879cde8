"""One profiled VQGAN encode of a 16-frame clip (after a warm-up) between cudaProfilerStart/Stop:
  ncu --profile-from-start off --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum --csv \
      --log-file x.csv python tools/prof_vqgan_once.py [frames] [precision]"""
import os
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from lwm_b200.vqgan import VQGAN, init_params
n = int(sys.argv[1]) if len(sys.argv) > 1 else 16
prec = sys.argv[2] if len(sys.argv) > 2 else "fp16x2"
tok = VQGAN(init_params(seed=0), precision=prec)
g = torch.Generator().manual_seed(1234)
x = (torch.rand(n, 256, 256, 3, generator=g) * 2 - 1).cuda()
tok.encode(x)
torch.cuda.synchronize()
torch.cuda.profiler.start()
tok.encode(x)
torch.cuda.synchronize()
torch.cuda.profiler.stop()
print("profiled one encode of %d frames (%s)" % (n, prec))
