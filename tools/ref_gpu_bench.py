"""Library bar (SURVEY.md section 8d): the UNMODIFIED reference's own --devices cuda:0 path (cuDNN / cuBLAS, TF32 off by
torch default for matmul, cuDNN conv TF32 on) timed on the same synthetic workload as bench.py.
Needs the reference modules under oracle/_ref (copied by build() where a reference checkout is present).  Usage: python tools/ref_gpu_bench.py [size] [iters]"""
import json
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from oracle import reference_harness as RH  # noqa: E402
from oracle import st_oracle as O  # noqa: E402

size = int(sys.argv[1]) if len(sys.argv) > 1 else 2048
iters = int(sys.argv[2]) if len(sys.argv) > 2 else 20
wts = O.make_vgg_weights(1234)
content, style = O.synth_image(1, 16, size, size), O.synth_image(2, 32, size, size)
t, trace = RH.time_reference(size, iters, wts, content, style, devices=('cuda:0',), skip=3)
print(json.dumps(dict(impl='reference-cuda', size=size, iters=iters, s_per_it=t, it_per_s=1.0 / t,
                      final_loss=trace[-1]['loss'], gpu=torch.cuda.get_device_name(0),
                      max_mem_gb=torch.cuda.max_memory_allocated() / 2**30,
                      cudnn_allow_tf32=torch.backends.cudnn.allow_tf32,
                      matmul_allow_tf32=torch.backends.cuda.matmul.allow_tf32)))
