"""CLIP evaluation, CPU side: the fp32 oracle against the reference golden (tests/golden/clip_vitb32.pt, made by oracle/make_clip_golden.py
from the reference's own CLIP/clip/model.py), the host resize tables against Pillow bit for bit, state-dict / TorchScript loading and the
refusals."""
import os

import numpy as np
import pytest
import torch
from PIL import Image

from fatezero_b200 import clip_eval
from oracle import clip_oracle as co

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "clip_vitb32.pt")


@pytest.fixture(scope="module")
def gold():
    return torch.load(GOLDEN, weights_only=False)


def _small_oracle():
    torch.manual_seed(0)
    m = co.ClipOracle(64, 64, 2, 128, 32, 77, 1000, 128, 2, 2)
    for k, v in m.state_dict().items():
        v.copy_(co.synth_clip_state_dict(0, {k: tuple(v.shape)})[k] if k != "logit_scale" else torch.tensor(4.6))
    return m.eval().requires_grad_(False)


def test_frames_and_weights_match_the_golden(gold):
    assert co.frames_sha256(co.synth_clip_frames()) == gold["frames_sha256"]
    with torch.device("meta"):
        shapes = {k: tuple(v.shape) for k, v in co.ClipOracle(*co.VITB32).state_dict().items()}
    assert shapes == gold["shapes"]


def test_oracle_reproduces_the_golden(gold):
    m = co.oracle_model(0)
    frames = co.synth_clip_frames()
    pils = [co.crop_read(Image.fromarray(frames[k][i])) for k, i in gold["frame_order"]]
    px = torch.stack([co.preprocess(p) for p in pils])
    assert [co.array_sha256(p.numpy()) for p in px] == gold["pixels_sha256"]
    with torch.no_grad():
        img, txt = m.encode_image(px), m.encode_text(gold["ids"])
        logits = torch.stack([m(px, gold["ids"][list(p)])[0] for p in gold["pairs"]])
    for got, ref in ((img, gold["image_features"]), (txt, gold["text_features"]), (logits, gold["logits"])):
        assert (got - ref).abs().max().item() < 1e-4 * max(1.0, ref.abs().max().item())
    assert torch.equal(logits[..., 1] >= logits[..., 0], gold["success"])


SIZES = [(512, 512), (640, 360), (300, 500), (100, 150), (225, 224), (97, 1000), (333, 777), (1001, 223), (224, 225), (31, 17)]


@pytest.mark.parametrize("w,h", SIZES)
def test_resize_tables_equal_pillow(w, h):
    rng = np.random.default_rng(w * 1000 + h)
    img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    img[h // 3: h // 2] = 255  # saturated bands make the cubic's overshoot clip
    img[:, w // 4: w // 3] = 0
    size = clip_eval.resized_size(w, h)
    ref = np.asarray(Image.fromarray(img).resize(size, Image.BICUBIC))
    got = clip_eval.resample_numpy(img, size)
    assert got.shape == ref.shape and np.array_equal(got, ref)


def test_resize_matches_the_golden_resize(gold):
    frames = co.synth_clip_frames()
    got = []
    for k, i in gold["frame_order"]:
        im = np.asarray(co.crop_read(Image.fromarray(frames[k][i])))
        got.append(co.array_sha256(clip_eval.resample_numpy(im, clip_eval.resized_size(im.shape[1], im.shape[0]))))
    assert got == gold["resize_u8_sha256"]


def test_resized_size_and_frame_read():
    assert clip_eval.resized_size(640, 360) == (398, 224)
    assert clip_eval.resized_size(150, 100) == (336, 224)
    assert clip_eval.resized_size(360, 640) == (224, 398)
    assert clip_eval.frame_read_size(360, 640) == (360, 360)
    assert clip_eval.frame_read_size(640, 360) == (640, 360)


def test_parse_openai_layout_and_torchscript_archive(tmp_path):
    g = clip_eval.parse_state_dict(co.synth_clip_state_dict(0))
    assert (g["width"], g["patch"], g["grid"], g["resolution"], g["vision_layers"], g["vision_heads"]) == (768, 32, 7, 224, 12, 12)
    assert (g["embed_dim"], g["context_length"], g["vocab_size"], g["text_width"], g["text_layers"], g["text_heads"]) == (512, 77, 49408, 512, 12, 8)
    m = _small_oracle()
    ids = torch.zeros(2, 77, dtype=torch.long)
    ids[:, 0], ids[0, 5], ids[1, 9] = 998, 999, 999
    path = str(tmp_path / "ViT-test.pt")
    torch.jit.trace(m, (torch.randn(2, 3, 64, 64), ids), check_trace=False).save(path)
    sd = clip_eval.load_state_dict(path)
    assert set(sd) == set(m.state_dict()) and all(torch.equal(sd[k], v) for k, v in m.state_dict().items())
    g = clip_eval.parse_state_dict(sd)
    assert (g["width"], g["grid"], g["vision_layers"], g["text_layers"], g["embed_dim"]) == (128, 2, 2, 2, 64)
    plain = str(tmp_path / "plain.pt")
    torch.save(m.state_dict(), plain)
    assert set(clip_eval.load_state_dict(plain)) == set(sd)


def test_refusals():
    sd = _small_oracle().state_dict()
    resnet = {k: v for k, v in sd.items() if k != "visual.proj"}
    resnet["visual.layer1.0.conv1.weight"] = torch.zeros(1)
    with pytest.raises(NotImplementedError, match="ResNet"):
        clip_eval.parse_state_dict(resnet)
    rect = dict(sd)
    rect["visual.conv1.weight"] = torch.zeros(128, 3, 32, 16)
    with pytest.raises(NotImplementedError, match="square"):
        clip_eval.parse_state_dict(rect)
    for k in ("ln_final.weight", "transformer.resblocks.1.mlp.c_fc.bias"):
        with pytest.raises(KeyError, match=k.replace(".", r"\.")):
            clip_eval.parse_state_dict({kk: v for kk, v in sd.items() if kk != k})
    with pytest.raises(RuntimeError, match="CUDA"):
        clip_eval.ClipEvaluator(sd, device="cpu")


def test_score_batch_argument_checks():
    ev = clip_eval.ClipEvaluator.__new__(clip_eval.ClipEvaluator)  # the checks run before any device work
    with pytest.raises(ValueError, match="at least one clip"):
        ev.score_batch([], "a", [])
    x = torch.zeros(2, 8, 8, 3, dtype=torch.uint8)
    with pytest.raises(ValueError, match="2 clips but 1 target"):
        ev.score_batch([x, x], "a", ["b"])
    with pytest.raises(ValueError, match="1 clips but 2 target"):
        ev.score_batch([x], "a", ["b", "c"])


def test_tokenize_is_required_without_openai_clip(monkeypatch):
    import sys
    monkeypatch.delenv("FATEZERO_REFERENCE_ROOT", raising=False)
    monkeypatch.setitem(sys.modules, "clip", None)
    with pytest.raises(RuntimeError, match="tokenize="):
        clip_eval._default_tokenize()


def test_clip_kernels_do_not_spill(tmp_path):
    import re
    import shutil
    import subprocess
    from fatezero_b200 import _build
    nvcc = _build._nvcc()
    if not (os.path.isabs(nvcc) and os.path.exists(nvcc)) and not shutil.which(nvcc):
        pytest.skip("nvcc not available")
    src = os.path.join(_build.CSRC, "fz_clip.cu")
    out = subprocess.run([nvcc, *_build.NVCC_FLAGS, "-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "fz_clip.o")], capture_output=True,
                         text=True, check=True)
    log = out.stdout + out.stderr
    kernels = re.findall(r"Compiling entry function '(\w+)'", log)
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", log)
    assert len(kernels) == 7 and len(spills) == 7, log
    assert all(s == ("0", "0") for s in spills), log
