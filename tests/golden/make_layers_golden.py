"""Golden vectors of the layer attributes, from the UNMODIFIED reference on CPU (as make_golden.py, whose CASES stay
untouched so that no existing fixture is regenerated).

Run once in the build container:  python tests/golden/make_layers_golden.py [A B ...]
Writes tests/golden/layers_<name>.npz for each configuration below, with StyleTransfer.content_layers, style_layers and
style_weights set after construction, as a user would:
  single_losses / single_final   stylize() at 64x48, single scale, 6 iterations
  pyr_losses / pyr_sizes / pyr_final   stylize() 32 -> 64 (4 + 3 iterations)
  image / terms / total / grad   one closure on a perturbed 64x48 image: the per-term losses in SumLoss order (content
                                 terms, style terms, TV; ST:455) and d loss / d image from the reference's autograd
Fixture: VGG-19 conv weights = oracle.st_oracle.make_vgg_weights(1234), content (1, 16, 64, 48), style (2, 32, 56, 40),
max pooling, torch.manual_seed(0).
"""
import contextlib
import io
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
from oracle import reference_harness as R  # noqa: E402
from oracle import st_oracle as O  # noqa: E402

OUT = Path(__file__).resolve().parent

# name -> (content_layers, style_layers, style_weights as set on the object).  There is no fixture for an empty
# style_layers: the reference's stylize() raises ValueError on it (the style-image forward takes max() of the empty list,
# ST:63, 81, 440).
CONFIGS = {
    'A': ([11], [1, 6, 11], [w / 341 for w in (256, 64, 16, 4, 1)]),
    'B': ([22], [1, 6, 11, 20, 22, 29], [w / 345 for w in (256, 64, 16, 4, 4, 1)]),
    'C': ([1, 29], [20], [w / 341 for w in (256, 64, 16, 4, 1)]),
    'E': ([22], [1, 6], [w / 341 for w in (256, 64, 16, 4, 1)]),
}
CONTENT, STYLE = (1, 16, 64, 48), (2, 32, 56, 40)
SINGLE = dict(min_scale=64, end_scale=64, initial_iterations=6)
PYRAMID = dict(min_scale=32, end_scale=64, iterations=3, initial_iterations=4)


def make_reference(ref, weights, name):
    content_layers, style_layers, style_weights = CONFIGS[name]
    torch.manual_seed(0)
    with R.patched_checkpoint(weights):
        st = ref.StyleTransfer(devices=['cpu'], pooling='max')
    st.content_layers, st.style_layers, st.style_weights = list(content_layers), list(style_layers), list(style_weights)
    return st


def run(ref, weights, name, kw):
    st = make_reference(ref, weights, name)
    trace = []
    with contextlib.redirect_stdout(io.StringIO()):
        st.stylize(O.synth_image(*CONTENT), [O.synth_image(*STYLE)],
                   callback=lambda it: trace.append((it.loss, it.w, it.h, it.i)), **kw)
    return (np.array([t[0] for t in trace], dtype=np.float64), np.array([t[1:] for t in trace], dtype=np.int32),
            st.get_image_tensor().numpy().astype(np.float32))


def internals(ref, weights, name):
    """One closure as stylize() builds it (ST:425-476), on a perturbed image."""
    from PIL import Image
    st = make_reference(ref, weights, name)
    content, style = O.synth_image(*CONTENT), O.synth_image(*STYLE)
    cw, ch = 64, 48
    cimg = ref.TF.to_tensor(content.resize((cw, ch), Image.BICUBIC))[None]
    simg = ref.TF.to_tensor(style.resize(ref.size_to_fit(style.size, 64), Image.BICUBIC))[None]
    g = torch.Generator().manual_seed(123)
    img = (cimg + 0.05 * torch.randn(cimg.shape, generator=g)).clamp(0, 1).requires_grad_()
    content_weights = [0.015 / len(st.content_layers)] * len(st.content_layers)
    feats_c = st.model(cimg, layers=st.content_layers)
    losses = [ref.Scale(ref.LayerApply(ref.ContentLossMSE(feats_c[layer]), layer), w)
              for layer, w in zip(st.content_layers, content_weights)]
    if st.style_layers:
        sfeats = st.model(simg, layers=st.style_layers)
        for layer, w in zip(st.style_layers, st.style_weights):
            losses.append(ref.Scale(ref.LayerApply(ref.StyleLossW2(ref.StyleLossW2.get_target(sfeats[layer])), layer),
                                    w))
    losses.append(ref.Scale(ref.LayerApply(ref.TVLoss(), 'input'), 2.0))
    feats = st.model(img)
    terms = [loss(feats) for loss in losses]
    total = sum(terms)
    total.backward()
    return img.detach().numpy(), np.array([float(t) for t in terms]), float(total), img.grad.numpy()


def main():
    weights = O.make_vgg_weights(1234)
    ref = R.import_reference()
    only = set(sys.argv[1:])
    for name in CONFIGS:
        if only and name not in only:
            continue
        s_losses, _, s_final = run(ref, weights, name, SINGLE)
        p_losses, p_sizes, p_final = run(ref, weights, name, PYRAMID)
        image, terms, total, grad = internals(ref, weights, name)
        np.savez_compressed(OUT / f'layers_{name}.npz', single_losses=s_losses, single_final=s_final,
                            pyr_losses=p_losses, pyr_sizes=p_sizes, pyr_final=p_final, image=image, terms=terms,
                            total=total, grad=grad)
        print(name, s_losses[:2], p_losses[-1], terms, flush=True)


if __name__ == '__main__':
    main()
