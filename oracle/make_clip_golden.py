"""Generate tests/golden/clip_vitb32.pt by running the UNMODIFIED reference CLIP (CLIP/clip/model.py `CLIP`, CLIP/clip/clip.py `_transform`
and `tokenize`) on the CPU in fp32, with the synthetic ViT-B/32 weights and frames of oracle/clip_oracle.py.  Needs the reference checkout
(FZ_REFERENCE_ROOT, default /root/reference); the tokenizer's ftfy import is served by oracle/shim/ftfy.
Usage: python -m oracle.make_clip_golden"""
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import clip_oracle as co  # noqa: E402
from oracle.ref_harness import REFERENCE_ROOT, _SHIM  # noqa: E402


def main():
    import yaml
    from PIL import Image
    for p in (_SHIM, os.path.join(REFERENCE_ROOT, "CLIP")):
        sys.path.insert(0, p)
    import clip as ref_clip
    from clip.model import CLIP

    t0 = time.time()
    torch.manual_seed(0)
    model = CLIP(*co.VITB32).eval().requires_grad_(False)
    shapes = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    model.load_state_dict(co.synth_clip_state_dict(0, shapes))
    preprocess = ref_clip.clip._transform(224)

    bench = yaml.safe_load(open(os.path.join(REFERENCE_ROOT, "CLIP", "bench_clean_prompt.yaml")))
    names = list(bench)
    prompts = []
    for n in names:
        for s in (bench[n]["source"], bench[n]["target"]):
            if s not in prompts:
                prompts.append(s)
    ids = ref_clip.tokenize(prompts).long()

    frames = co.synth_clip_frames()
    order = [(k, i) for k in sorted(frames) for i in range(frames[k].shape[0])]
    pils = [co.crop_read(Image.fromarray(frames[k][i])) for k, i in order]
    pixels = torch.stack([preprocess(p) for p in pils])
    resize = preprocess.transforms[0]

    with torch.no_grad():
        img = model.encode_image(pixels)
        txt = model.encode_text(ids)
        pairs = [(prompts.index(bench[n]["source"]), prompts.index(bench[n]["target"])) for n in names]
        logits = torch.stack([model(pixels, ids[list(p)])[0] for p in pairs])           # [E, images, 2]
    probs = logits.softmax(-1)
    success = probs[..., 1] >= probs[..., 0]
    sel = [j for j, (k, _) in enumerate(order) if k == "clip512"]
    nf = img[sel] / torch.sqrt(torch.sum(img[sel] ** 2, axis=1, keepdims=True))
    cos = torch.stack([torch.sum(nf[i] * nf[i + 1]) for i in range(len(sel) - 1)])
    gold = dict(
        shapes=shapes, seed=0, logit_scale=float(model.logit_scale.detach()), frames_sha256=co.frames_sha256(frames),
        frame_order=order, prompt_names=names, prompts=prompts, ids=ids, pairs=pairs,
        # the preprocess outputs of every image, as digests of their bytes (bitwise checks without storing the pixels)
        resize_u8_sha256=[co.array_sha256(np.asarray(resize(p))) for p in pils],
        pixels_sha256=[co.array_sha256(px.numpy()) for px in pixels],
        image_features=img.clone(), text_features=txt.clone(), logits=logits.clone(), probs=probs.clone(), success=success.clone(),
        clip512_cosines=cos.clone(), clip512_consistency=float(cos.sum() / len(cos)), seconds=time.time() - t0, torch=str(torch.__version__))
    path = os.path.join(ROOT, "tests", "golden", "clip_vitb32.pt")
    torch.save(gold, path)
    print(path, f"{os.path.getsize(path) / 1e6:.2f} MB", f"{gold['seconds']:.1f}s", f"{len(prompts)} prompts, {len(order)} images",
          f"success rate {success.float().mean():.3f}, min |margin| {(logits[..., 1] - logits[..., 0]).abs().min():.4f}")


if __name__ == "__main__":
    main()
