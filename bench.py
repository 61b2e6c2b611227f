#!/usr/bin/env python
"""Benchmark of the stylize() hot path: iterations/sec at end_scale=2048 (BASELINE.json metric).

  python bench.py [--gpus N] [--steps K] [--warmup W] [--size 2048] [--impl native|reference] [--dump-outputs DIR]

A "step" is one stylize iteration (VGG-19 forward, W2/content/TV losses, backward to the image, Adam+clamp+EMA)
on a synthetic 2048x2048 content+style pair with the seeded synthetic VGG-19 (no network for images/checkpoints).

native arm   value   = it/s of K stb_iterate calls, state resident in HBM, CUDA events on the launching stream,
                       barrier + synchronize on both sides, max over ranks.
             e2e     = it/s of the public API: StyleTransfer.stylize(PIL content, [PIL style], single scale, K
                       iterations, callback reading the loss every iteration) -- host PIL inputs, H2D of the
                       resized images, per-iteration D2H of the loss, final D2H of the result, all inside the timed
                       region (wall clock around the call, since it spans host work).
             roofline= conv tensor-pipe: algorithmic conv FLOPs per iteration / summed duration of the wgmma conv
                       launches (CUDA events around every launch, second instrumented pass), vs the bf16 peak of
                       MEASURED_PEAKS.json, else the H100 SXM data sheet's dense bf16 figure.
             cpu_baseline = the UNMODIFIED reference (oracle/_ref; else the oracle port) timed on all host cores for one
                       real iteration at the benchmark size after a warm-up iteration (no extrapolation).
--dump-outputs DIR: after the timed steps, rank 0 writes what the last timed step computed -- the image, the EMA of
                       the image and the eight loss values -- as DIR/<name>.npy (float32, at most 64 MB in all; an array
                       over its share is written as a fixed, seeded sample <name>_sample.npy).  The inputs depend on
                       the arguments only, so two builds can be compared output for output.
reference arm (--impl reference): 2-3 real 2048^2 iterations of the reference's CPU path + configs[0] (256^2, 50
                       iterations), printed in the same JSON shape.
N > 1: ONE 2048x2048 job tiled spatially over the N GPUs (strong scaling): horizontal bands with 80-row halo aprons;
per iteration one all-reduce of the 2.4 MB statistics block, a seam reduce of the image gradient (fused with Adam)
and a halo pull, all as kernels reading the peers' mailboxes over NVLink inside ONE CUDA graph per rank
(style-transfer-pytorch_b200/csrc/comm.cu, distributed.py; SURVEY.md section 8e).  The line then carries
`parity_vs_n1`: the tiled loss trace against rank 0's untiled run of the same job.
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent
sys.path.insert(0, str(ROOT))

CONV_FLOP_PER_PIXEL = 1444608.0  # fwd + dgrad, 2 flop/MAC (SURVEY.md section 8d)
CONV0_FLOP_PER_PIXEL = 4 * 27 * 64.0  # conv0 fwd + dgrad run in their own kernels (conv0_tc.cu), not in the timed class
PROF_CLASSES = ['conv0_fwd_tv', 'conv_fwd', 'pool_fwd', 'gram', 'sse', 'w2', 'conv_bwd', 'pool_bwd',
                'conv0_bwd_adam', 'finalize']


def measured_peaks():
    p = ROOT / 'MEASURED_PEAKS.json'
    if p.exists():
        d = json.loads(p.read_text())
        return dict(hbm_gbs=d['hbm_gbs'], bf16_tflops=d['bf16_tflops'],
                    bf16_tflops_sustained=d.get('bf16_tflops_sustained', d['bf16_tflops']), source='measured')
    # NVIDIA H100 SXM data sheet (700 W): 3.35 TB/s HBM3, 989 TFLOP/s dense bf16 -- a ceiling, not a measured rate
    return dict(hbm_gbs=3350.0, bf16_tflops=989.0, bf16_tflops_sustained=989.0, source='H100 SXM data sheet')


def dump_outputs(out_dir, arrays, budget=64 << 20):
    """Write each (name, tensor, share of the byte budget) as out_dir/<name>.npy in float32; a tensor larger than its
    share is written as <name>_sample.npy, the elements at a fixed, seeded set of flat indices."""
    import numpy as np
    out_dir.mkdir(parents=True, exist_ok=True)
    for name, t, share in arrays:
        a = t.detach().float().cpu().numpy()
        cap = int(budget * share) // 4
        if a.size <= cap:
            np.save(out_dir / f'{name}.npy', a)
        else:
            idx = np.sort(np.random.default_rng(0).choice(a.size, cap, replace=False))
            np.save(out_dir / f'{name}_sample.npy', a.ravel()[idx])


class ClockSampler:
    """nvidia-smi clocks / throttle reasons during the timed region."""
    Q = ('index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,'
         'clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,'
         'clocks_event_reasons.sw_power_cap')

    def __init__(self, gpu_index):
        self.gpu = gpu_index
        self.proc = None
        self.lines = []

    def start(self):
        try:
            self.proc = subprocess.Popen(['nvidia-smi', '-i', str(self.gpu), f'--query-gpu={self.Q}',
                                          '--format=csv,noheader,nounits', '-lms', '100'],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.thread = threading.Thread(target=self._read, daemon=True)
            self.thread.start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.lines.append(line.strip())

    def stop(self):
        if self.proc is None:
            return dict(sm_mhz=None, sm_max_mhz=None, reasons=['nvidia-smi unavailable'])
        self.proc.terminate()
        try:
            self.proc.wait(timeout=2)
        except Exception:
            self.proc.kill()
        sm, smax, reasons = [], None, set()
        names = ['hw_slowdown', 'hw_thermal_slowdown', 'sw_thermal_slowdown', 'sw_power_cap']
        for line in self.lines:
            parts = [x.strip() for x in line.split(',')]
            if len(parts) < 8:
                continue
            try:
                sm.append(float(parts[1]))
                smax = float(parts[2])
            except ValueError:
                continue
            for nm, val in zip(names, parts[4:8]):
                if val.lower().startswith('active'):
                    reasons.add(nm)
        sm.sort()
        hi = [v for v in sm if smax and v > 0.3 * smax] or sm
        med = hi[len(hi) // 2] if hi else None
        return dict(sm_mhz=med, sm_max_mhz=smax, reasons=sorted(reasons), samples=len(sm))


# ------------------------------------------------------------------------------------------------ CPU baseline
def _use_all_host_threads():
    """torchrun exports OMP_NUM_THREADS=1: the CPU arm must still use every host core (the reference's CPU path does)."""
    import torch
    try:
        import psutil
        n = psutil.cpu_count(logical=False) or os.cpu_count() or 1   # physical cores: SMT siblings slow oneDNN down
    except Exception:
        n = max(1, (os.cpu_count() or 2) // 2)
    if torch.get_num_threads() != n:
        torch.set_num_threads(n)
    return torch.get_num_threads()


class _Budget(Exception):
    pass


def reference_iteration_times(size, n_iters, budget_s):
    """Per-iteration wall times of the UNMODIFIED reference's stylize() (single scale, size x size, CPU) when build()
    copied it into oracle/_ref, else of the oracle port of the same loop body.  Returns
    (kind, [seconds per iteration, first one excluded], threads).  Stops early once budget_s is exceeded."""
    import torch
    from oracle import reference_harness as RH
    from oracle import st_oracle as O
    threads = _use_all_host_threads()
    wts = O.make_vgg_weights(1234)
    content, style = O.synth_image(1, 16, size, size), O.synth_image(2, 32, size, size)
    stamps = []
    t_start = time.perf_counter()
    if RH.reference_available():
        kind = 'reference'
        ref = RH.import_reference()

        def cb(it):
            stamps.append(it.time)   # ST:493
            if len(stamps) >= 2 and time.perf_counter() - t_start > budget_s:
                raise _Budget()

        torch.manual_seed(0)
        with RH.patched_checkpoint(wts):
            st = ref.StyleTransfer(devices=['cpu'], pooling='max')
        import contextlib
        import io
        try:
            with contextlib.redirect_stdout(io.StringIO()):
                st.stylize(content, [style], min_scale=size, end_scale=size, initial_iterations=n_iters + 1, callback=cb)
        except _Budget:
            pass
    else:
        kind = 'port'
        tg, _ = O.make_targets(content, [style], [1.0], size, wts, 'max', 0.015, 2.0)
        state = O.IterState.fresh(O.to_tensor(content))
        for _ in range(n_iters + 1):
            O.iterate(state, wts, tg, 'max')
            stamps.append(time.time())
            if len(stamps) >= 2 and time.perf_counter() - t_start > budget_s:
                break
    return kind, [b - a for a, b in zip(stamps[:-1], stamps[1:])], threads


def cpu_baseline(size, n_iters=1, budget_s=90.0):
    """The reference's CPU path on the host cores, REAL iterations at the benchmark size (no extrapolation)."""
    kind, dts, threads = reference_iteration_times(size, n_iters, budget_s)
    dts = sorted(dts)
    med = dts[len(dts) // 2]
    what = ('unmodified reference StyleTransfer.stylize(devices=[cpu])' if kind == 'reference'
            else 'oracle port (torch-CPU explicit schedule)')
    return dict(value=1.0 / med, unit='it/s', cores=threads, kind=kind,
                sample=f'{what}: {len(dts)} timed iteration(s) at {size}x{size} after one warm-up iteration, '
                       f'median {med:.2f} s/it (all: {[round(d, 2) for d in dts]})')


# ------------------------------------------------------------------------------------------------ arms
def run_reference(args, rank, world):
    if rank != 0:
        return
    # a bounded sample of the SAME workload: real 2048^2 iterations of the reference on all host threads
    n = max(2, min(args.steps, 3))
    cb = cpu_baseline(args.size, n_iters=n, budget_s=150.0)
    # BASELINE.json configs[0]: 256 x 256, 50 iterations, single scale, --devices cpu
    kind0, d0, _ = reference_iteration_times(256, 50, 60.0)
    d0 = sorted(d0)
    line = dict(metric='stylize iterations/sec at end_scale=2048', value=cb['value'], unit='it/s', n_gpus=args.gpus,
                steps=args.steps, warmup=args.warmup, ms_per_step=1000.0 / cb['value'], higher_is_better=True,
                scaling='strong', vs_baseline=None, dtype='f32', data='synthetic', impl='reference',
                config=dict(workload=f'{args.size}x{args.size} single scale, pooling=max, content+1 style, '
                                     'CPU reference path (' + cb['kind'] + '), real iterations at this size',
                            config0=dict(workload='256x256 single scale, 50 iterations (BASELINE.json configs[0])',
                                         kind=kind0, it_per_s=1.0 / d0[len(d0) // 2], iterations_timed=len(d0))),
                cpu_baseline=cb, e2e=dict(value=cb['value'], unit='it/s', h2d_bytes_per_step=0, d2h_bytes_per_step=0),
                gpu_launches=0)
    print(json.dumps(line), flush=True)


def run_native(args, rank, local_rank, world):
    import torch
    import torch.distributed as dist
    import ctypes
    import style_transfer_b200 as stb
    from style_transfer_b200 import _lib
    from oracle import st_oracle as O  # fixture generator (weights / synthetic images) + cpu_baseline leg only

    torch.cuda.set_device(local_rank)
    dev = torch.device('cuda', local_rank)
    # exactly ONE line on stdout: libraries (NCCL's version banner, torchrun) print there too, so fd 1 is pointed at
    # stderr for the duration of the run and the JSON line goes to the saved descriptor
    sys.stdout.flush()
    json_fd = os.dup(1)
    os.dup2(2, 1)
    if world > 1:
        dist.init_process_group('nccl', device_id=dev)
    size = args.size
    wts = O.make_vgg_weights(1234)
    content, style = O.synth_image(1, 16, size, size), O.synth_image(2, 32, size, size)
    from style_transfer_b200 import distributed as D
    st = stb.StyleTransfer(devices=[str(dev)], pooling='max', vgg_weights=wts)
    m = st.model
    band = D.make_band(size, rank, world) if world > 1 else None
    h_loc = band.h_local if band is not None else size
    cimg_full = O.to_tensor(content).to(dev)
    simg = O.to_tensor(style).to(dev)
    sband = D.make_band(size, rank, world) if world > 1 else None
    ws_sizes = [(h_loc, size), (sband.h_local if sband is not None else size, size)]
    if band is not None:   # mailboxes + (halo mode) the peer-mapped workspace, before anything touches the workspace
        st._ensure_peer_memory(ws_sizes, max(b.h_local for b in D.all_bands(size, world)), size)
    m.ensure_workspace(ws_sizes)
    means, srms = st._style_stats(simg, size, size)   # tiled over the ranks like the iterate when world > 1
    cimg = cimg_full
    if band is not None:
        cimg = D.local_slice(cimg_full, band)
        m.set_band(True, size, band.own0, band.own_rows)
    ct = m.content_features(cimg)
    m.set_targets(h_loc, size, ct, 0.015, means, srms, st.style_weights, 2.0)
    if band is not None:
        st._setup_comm(band, size)
    st.image = cimg.clone()
    st.average = stb.style_transfer.EMA(st.image, 0.99)
    ea, eas = torch.zeros_like(st.image), torch.zeros_like(st.image)
    step = 0
    stats = grad = None
    if band is not None and st._comm_mode != 'peer':
        stats, grad = m.stats_view(h_loc, size), torch.empty_like(st.image)

    def one_iteration():
        nonlocal step
        step += 1
        if band is not None:
            st._iterate_banded(band, stats, grad, ea, eas, step, 0.02, 0.99)
        else:
            st._iterate(ea, eas, step, 0.02, 0.99, True)

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    side = torch.cuda.Stream(device=dev)  # non-legacy stream: lets the library replay iterations as a CUDA graph
    side.wait_stream(torch.cuda.current_stream(dev))
    torch.cuda.set_stream(side)
    # ---- warm-up; the first PARITY_ITS of it double as the multi-GPU parity check (loss read back every iteration)
    PARITY_ITS = 5
    head = []
    for i in range(max(args.warmup, 3, PARITY_ITS)):
        one_iteration()
        if i < PARITY_ITS:
            side.synchronize()
            head.append(float(st._loss_host[0]))
    barrier()
    sampler = ClockSampler(local_rank)
    if rank == 0:
        sampler.start()
    # ---- REPEATS timed regions of exactly `steps` iterations each (barrier + synchronize on both sides, CUDA events,
    # max over ranks per region); the reported value is the MEDIAN region, the others are listed
    # (N = 1: a single region of exactly `steps` iterations; N > 1: five, because a tiled region of ~50 ms
    # is bimodal when any rank's host stalls)
    REPEATS = 5 if world > 1 else 1
    region_ms = []
    r0, k0, _ = m.launch_count()
    for _ in range(REPEATS):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        barrier()
        e0.record()
        for _ in range(args.steps):
            one_iteration()
        e1.record()
        barrier()
        t = torch.tensor([e0.elapsed_time(e1)], device=dev)
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        region_ms.append(float(t.item()))
    r1, k1, per_graph = m.launch_count()
    clocks = sampler.stop() if rank == 0 else None
    final_loss = float(st._loss_host[0])
    if args.dump_outputs and rank == 0:
        dump_outputs(Path(args.dump_outputs), [('image', st.image, 0.75), ('average', st.average.value, 0.15),
                                               ('loss_terms', st._loss_host, 0.05)])
    ms_total = sorted(region_ms)[len(region_ms) // 2]
    ms_per_step = ms_total / args.steps
    tiled = band is not None
    # tiled: all ranks advanced ONE job by `steps` iterations; otherwise (N == 1) the single job
    value = args.steps / (ms_total / 1000.0)
    # kernels launched inside the timed regions of THIS rank, counted from the captured graphs' kernel nodes
    launches_per_step = (k1 - k0) / max(1, REPEATS * args.steps)
    graph_ok, graph_note = m.graph_status()

    # ---- multi-GPU parity: rank 0 re-runs the first iterations of the SAME job untiled on its own GPU
    parity = None
    if tiled:
        if rank == 0:
            st1 = stb.StyleTransfer(devices=[str(dev)], pooling='max', vgg_weights=wts, distributed=False)
            m1 = st1.model
            m1.ensure_workspace([(size, size)])
            mm, ss = m1.style_stats(simg)
            ct1 = m1.content_features(cimg_full)
            m1.set_targets(size, size, ct1, 0.015, mm, ss, st1.style_weights, 2.0)
            st1.image = cimg_full.clone()
            st1.average = stb.style_transfer.EMA(st1.image, 0.99)
            a1, b1 = torch.zeros_like(st1.image), torch.zeros_like(st1.image)
            ref_head = []
            for i in range(PARITY_ITS):
                st1._iterate(a1, b1, i + 1, 0.02, 0.99, True)
                torch.cuda.current_stream().synchronize()
                ref_head.append(float(st1._loss_host[0]))
            rel = [abs(a - b) / abs(b) for a, b in zip(head, ref_head)]
            parity = dict(iterations=PARITY_ITS, tiled_losses=head, single_gpu_losses=ref_head,
                          max_rel_diff=max(rel), ok=max(rel) < 5e-4,
                          note='loss trace of the N-way tiled run vs the untiled run of the same job on rank 0')
            del st1, m1
            torch.cuda.empty_cache()
        barrier()

    # ---- instrumented pass: per-kernel-class device time (events around every launch; graphs off while profiling).
    # Tiled: every rank iterates (the exchanges need all of them), rank 0 records.
    prof = None
    n_prof = min(args.steps, 10)
    if rank == 0:
        _lib.check(m.lib.stb_profile_enable(m.ctx, 1))
    for _ in range(n_prof):
        one_iteration()
    torch.cuda.synchronize()
    if rank == 0:
        ms = (ctypes.c_float * 10)()
        cnt = (ctypes.c_int * 10)()
        _lib.check(m.lib.stb_profile_read(m.ctx, ms, cnt, 10))
        _lib.check(m.lib.stb_profile_enable(m.ctx, 0))
        prof = {name: dict(ms_per_iter=ms[i] / n_prof, launches_per_iter=cnt[i] / n_prof)
                for i, name in enumerate(PROF_CLASSES)}
    barrier()

    # ---- e2e through the public API (host PIL in, loss read back every iteration, result image on the host)
    e2e = None
    losses = []
    st2 = stb.StyleTransfer(devices=[str(dev)], pooling='max', vgg_weights=wts)
    import contextlib
    import io
    with contextlib.redirect_stdout(io.StringIO()):  # stylize() prints progress like the reference does
        st2.stylize(content, [style], min_scale=size, end_scale=size, initial_iterations=2, callback=lambda it: None)
    barrier()
    e2e_its = args.steps
    t0 = time.perf_counter()
    with contextlib.redirect_stdout(io.StringIO()):
        out = st2.stylize(content, [style], min_scale=size, end_scale=size, initial_iterations=e2e_its,
                          callback=lambda it: losses.append(it.loss))
    _ = out.size
    torch.cuda.synchronize()
    t_e2e = time.perf_counter() - t0
    te = torch.tensor([t_e2e], device=dev)
    if world > 1:
        dist.all_reduce(te, op=dist.ReduceOp.MAX)
    t_e2e = float(te.item())
    h2d = 2 * 3 * size * size                # content + style uint8 pixels (converted to fp32 on the device)
    d2h = 32 * e2e_its + 3 * size * size     # loss terms every step + final uint8 image
    e2e = dict(value=e2e_its / t_e2e, unit='it/s', h2d_bytes_per_step=h2d / e2e_its,
               d2h_bytes_per_step=d2h / e2e_its, iterations=e2e_its,
               note='StyleTransfer.stylize(PIL inputs, single scale, per-iteration loss callback) wall clock over '
                    f'{e2e_its} iterations, incl. PIL resize, target '
                    'extraction, H2D of the inputs, per-iteration loss D2H, final image D2H')

    if rank == 0:
        peaks = measured_peaks()
        # the twelve 3x3 convs of pixel_gemm_kernel on this rank's rows (band + aprons when tiled); the tap-gradient
        # GEMMs folded into the same launches (0.15 TFLOP at 2048^2) are NOT credited
        conv_flops = (CONV_FLOP_PER_PIXEL - CONV0_FLOP_PER_PIXEL) * h_loc * size
        conv_ms = prof['conv_fwd']['ms_per_iter'] + prof['conv_bwd']['ms_per_iter']
        achieved = conv_flops / (conv_ms / 1000.0) / 1e12
        peak = peaks['bf16_tflops_sustained']
        roofline = dict(bound='tensor', achieved=achieved, peak=peak, unit='TFLOP/s', frac=achieved / peak,
                        peak_source=f"{peaks['source']} (bf16_tflops_sustained)",
                        frac_of_burst_peak=achieved / peaks['bf16_tflops'],
                        kernel='pixel_gemm_kernel (wgmma conv fwd+dgrad incl. tap-gradient GEMMs, 25 launches/iter)',
                        note='algorithmic FLOPs/iter of the twelve 3x3 convs (1437696/pixel) / summed CUDA-event duration of the conv '
                             'launches in an instrumented pass of this run',
                        step_fraction=conv_ms / sum(v['ms_per_iter'] for v in prof.values()),
                        classes_ms_per_iter={k: round(v['ms_per_iter'], 4) for k, v in prof.items()},
                        whole_step_tensor_frac=CONV_FLOP_PER_PIXEL * size * size * (1000.0 / ms_per_step) / 1e12 /
                        (peak * world))
        cb = None
        if not args.no_cpu_baseline and world == 1:  # reported baseline: rank 0, N = 1 only
            cb = cpu_baseline(size, n_iters=1, budget_s=60.0)
        par = 'single GPU'
        if tiled:
            par = (f'{world}-way spatial tiling: bands of {band.own_rows}+{band.top_apron + band.bottom_apron} halo rows '
                   f'(rank 0); exchanges = ' +
                   ((f'peer-memory kernels inside the iteration graph, tile mode {"halo" if st._halo_now else "apron"} '
                     '(halo: own rows only + one boundary-row pull per layer; apron: 80 recomputed rows per side) '
                     '+ stats all-reduce, Adam on own rows, image halo pull; CUDA IPC over NVLink')
                    if st._comm_mode == 'peer' else
                    'host-driven NCCL (1 all-reduce + 2 send/recv per iteration)'))
        line = dict(metric='stylize iterations/sec at end_scale=2048', value=value, unit='it/s', n_gpus=world,
                    steps=args.steps, warmup=max(args.warmup, 3, PARITY_ITS), ms_per_step=ms_per_step,
                    higher_is_better=True, scaling='strong', vs_baseline=None, dtype='bf16', data='synthetic',
                    impl='native',
                    config=dict(workload=f'{size}x{size} single scale (BASELINE.json configs[2]), pooling=max, '
                                         'content+1 style, bf16 operands / fp32 accumulate, fp32 sqrtm+Adam',
                                parallelism=par,
                                l2='working set per iteration (>= 2.4 GB of activations) far exceeds the 50 MB L2',
                                final_loss=final_loss,
                                timing=(f'median of {REPEATS} timed regions of {args.steps} iterations each' if REPEATS > 1 else
                                        f'one timed region of {args.steps} iterations'),
                                regions_ms=[round(x, 3) for x in region_ms]),
                    clocks=clocks, e2e=e2e,
                    gpu_launches=int(round(launches_per_step * args.steps)),
                    gpu_launches_note=f'{launches_per_step:.1f} kernels per iteration, counted from the kernel nodes of '
                                      f'the replayed CUDA graph (per graph slot: {per_graph}); graph replay '
                                      f'{"on" if graph_ok == 1 else "OFF: " + graph_note}',
                    roofline=roofline, cpu_baseline=cb)
        if parity is not None:
            line['parity_vs_n1'] = parity
        sys.stdout.flush()
        os.write(json_fd, (json.dumps(line) + '\n').encode())
    if world > 1:
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--gpus', type=int, default=1)
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--size', type=int, default=2048)
    ap.add_argument('--impl', default='native', choices=['native', 'reference'])
    ap.add_argument('--no-cpu-baseline', action='store_true')
    ap.add_argument('--dump-outputs', metavar='DIR', default=None)
    args = ap.parse_args()
    rank = int(os.environ.get('RANK', '0'))
    local_rank = int(os.environ.get('LOCAL_RANK', '0'))
    world = int(os.environ.get('WORLD_SIZE', '1'))
    if args.impl == 'reference':
        run_reference(args, rank, world)
    else:
        run_native(args, rank, local_rank, world)


if __name__ == '__main__':
    main()
