"""TEST / BASELINE INFRASTRUCTURE ONLY -- runs the UNMODIFIED reference with the synthetic VGG fixture.

The reference modules are looked up in oracle/_ref (git-ignored; `build()` copies them there from a reference checkout
when one is present: oracle/Makefile's default location or STB_REFERENCE_DIR).  Used by tests/golden/make_golden.py to produce the committed golden vectors that pin
oracle/st_oracle.py, by tests that are skipped when the reference is absent, and by bench.py's reference arm /
cpu_baseline leg.  The only thing patched is torchvision's checkpoint *download* (no network needed): the reference
code itself runs untouched.
"""
from __future__ import annotations

import contextlib
import io
import sys
from pathlib import Path

import torch

REFERENCE_ROOT = Path(__file__).resolve().parent / '_ref'


def reference_available() -> bool:
    return (REFERENCE_ROOT / 'style_transfer' / 'style_transfer.py').exists()


def _full_vgg_state_dict(conv_weights):
    """state_dict for torchvision vgg19 with our conv weights; classifier (unused: ST:35 keeps .features[:30]) zero."""
    from torchvision import models
    conv_idx = [0, 2, 5, 7, 10, 12, 14, 16, 19, 21, 23, 25, 28, 30, 32, 34]
    sd = {}
    full = models.vgg19(weights=None)
    for k, v in full.state_dict().items():
        sd[k] = torch.zeros_like(v)
    for (w, b), i in zip(conv_weights, conv_idx):
        sd[f'features.{i}.weight'] = w.clone()
        sd[f'features.{i}.bias'] = b.clone()
    return sd


@contextlib.contextmanager
def patched_checkpoint(conv_weights):
    """Serve the synthetic VGG-19 state_dict in place of the ImageNet download (vgg19-dcbb9e9d.pth)."""
    import torchvision.models._api as api
    sd = _full_vgg_state_dict(conv_weights)
    orig = api.load_state_dict_from_url
    api.load_state_dict_from_url = lambda *a, **k: sd
    try:
        yield
    finally:
        api.load_state_dict_from_url = orig


def import_reference():
    """Import the reference's style_transfer.style_transfer module without its package __init__ (which pulls the
    aiohttp web UI); the module itself is loaded unmodified."""
    import importlib.util
    import types
    name = 'ref_style_transfer'
    if name + '.style_transfer' in sys.modules:
        return sys.modules[name + '.style_transfer']
    pkg = types.ModuleType(name)
    pkg.__path__ = [str(REFERENCE_ROOT / 'style_transfer')]
    sys.modules[name] = pkg
    for sub in ('sqrtm', 'style_transfer'):
        spec = importlib.util.spec_from_file_location(f'{name}.{sub}', REFERENCE_ROOT / 'style_transfer' / f'{sub}.py')
        mod = importlib.util.module_from_spec(spec)
        sys.modules[f'{name}.{sub}'] = mod
        spec.loader.exec_module(mod)
        setattr(pkg, sub, mod)
    return sys.modules[name + '.style_transfer']


def run_reference(content_pil, style_pils, conv_weights, pooling='max', seed=0, quiet=True, devices=('cpu',),
                  **stylize_kwargs):
    """Run reference StyleTransfer.stylize(); returns (final PIL-free image tensor, trace, st)."""
    ref = import_reference()
    trace = []

    def cb(it):
        trace.append(dict(w=it.w, h=it.h, i=it.i, i_max=it.i_max, loss=it.loss, time=it.time))

    torch.manual_seed(seed)
    with patched_checkpoint(conv_weights):
        st = ref.StyleTransfer(devices=list(devices), pooling=pooling)
    out = io.StringIO()
    with contextlib.redirect_stdout(out if quiet else sys.stdout):
        st.stylize(content_pil, style_pils, callback=cb, **stylize_kwargs)
    return st.get_image_tensor(), trace, st


def time_reference(size, iters, conv_weights, content_pil, style_pil, devices=('cpu',), skip=2):
    """Seconds per iteration of the unmodified reference at size x size (single scale): median of the differences of
    STIterate.time (ST:493), the first `skip` iterations excluded."""
    _, trace, _ = run_reference(content_pil, [style_pil], conv_weights, devices=devices, min_scale=size,
                                end_scale=size, initial_iterations=iters + skip + 1)
    t = [r['time'] for r in trace]
    d = sorted(b - a for a, b in zip(t[skip:-1], t[skip + 1:]))
    return d[len(d) // 2], trace
