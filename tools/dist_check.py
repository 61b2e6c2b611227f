"""Multi-GPU check (run with torchrun, one rank per GPU): banded stylize() == single-GPU stylize().
  python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29511 \
      tools/dist_check.py [H W its [adam|lbfgs]]
With lbfgs the loss bar after the first stored pair is the one of tests/test_gpu_lbfgs_tiled.py (1e-2): L-BFGS
amplifies the ~1e-4 closure difference that the split statistics' summation order makes."""
import contextlib
import io
import os
import sys
import time
from pathlib import Path

import numpy as np
import torch
import torch.distributed as dist

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import style_transfer_b200 as stb  # noqa: E402
from oracle import st_oracle as O  # noqa: E402  (fixture generator only)

H = int(sys.argv[1]) if len(sys.argv) > 1 else 384
W = int(sys.argv[2]) if len(sys.argv) > 2 else 512
ITS = int(sys.argv[3]) if len(sys.argv) > 3 else 6
OPT = sys.argv[4] if len(sys.argv) > 4 else 'adam'
rank, local, world = int(os.environ['RANK']), int(os.environ['LOCAL_RANK']), int(os.environ['WORLD_SIZE'])
torch.cuda.set_device(local)
dist.init_process_group('nccl', device_id=torch.device('cuda', local))
wts = O.make_vgg_weights(1234)
content, style = O.synth_image(1, 16, W, H), O.synth_image(2, 32, W // 2 + 40, H // 2 + 24)
scale = max(H, W)
kw = dict(min_scale=scale, end_scale=scale, initial_iterations=ITS, optimizer=OPT)


MODES = []


def run(distributed):
    st = stb.StyleTransfer(devices=[f'cuda:{local}'], pooling='max', vgg_weights=wts, distributed=distributed)
    tr = []
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    with contextlib.redirect_stdout(io.StringIO()):
        img = st.stylize(content, [style], callback=lambda it: tr.append(it.loss), **kw)
    torch.cuda.synchronize()
    MODES.append(((st._comm_mode, 'halo' if st._halo_now else 'apron') if distributed is not False else 'single', st.model.graph_status()))
    return np.array(tr), np.asarray(img, dtype=np.float32), time.perf_counter() - t0


tr_b, img_b, t_b = run(None)
tr_s, img_s, t_s = run(False)
rel = np.abs(tr_b - tr_s) / np.abs(tr_s)
d = np.abs(img_b - img_s)
if OPT == 'lbfgs':   # before the first stored pair as Adam, after it L-BFGS amplifies the closure difference
    ok = rel[:2].max() < 5e-4 and rel.max() < 1e-2 and d.mean() < 5e-3 * 255
else:
    ok = rel.max() < 5e-4 and d.mean() < 0.5  # 1e-3 is the loss bar; summation order alone moves the loss by ~1e-4
print(f'[rank {rank}/{world}] banded {tr_b[:3]}..{tr_b[-1]:.6f} ({t_b:.2f}s) single {tr_s[:3]}..{tr_s[-1]:.6f} ({t_s:.2f}s) '
      f'{OPT}: max rel loss diff {rel.max():.2e}  image mean |diff| {d.mean():.3f}/255 max {d.max():.0f}  modes {MODES}  '
      f'{"OK" if ok else "BAD"}',
      flush=True)
flag = torch.tensor([int(ok)], device='cuda')
dist.all_reduce(flag, op=dist.ReduceOp.MIN)
dist.destroy_process_group()
sys.exit(0 if flag.item() == 1 else 1)
