"""CLIP text encoder on the sm_90a kernels (fatezero_b200/clip.py) against transformers' CLIPTextModel (the module the reference calls at
pipelines/stable_diffusion.py:230,279), same random-init weights, fp32 torch on the GPU as the checker.  Bound: fp16 storage through 12
layers vs fp32 — measured value printed, bound 2x."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _model(seed=0):
    from transformers import CLIPTextConfig, CLIPTextModel
    torch.manual_seed(seed)
    cfg = CLIPTextConfig(vocab_size=49408, hidden_size=768, intermediate_size=3072, num_hidden_layers=12, num_attention_heads=12,
                         max_position_embeddings=77, hidden_act="quick_gelu")
    return CLIPTextModel(cfg).eval().requires_grad_(False).cuda()


def test_clip_engine_matches_transformers(report):
    from fatezero_b200.clip import ClipTextEngine
    m = _model()
    ids = torch.randint(0, 49408, (2, 77), generator=torch.Generator().manual_seed(1)).cuda()
    ids[:, 0] = 49406
    ids[0, 12:] = 49407
    torch.backends.cuda.matmul.allow_tf32 = False
    ref = m(ids)[0].float()
    got = ClipTextEngine(m)(ids)[0]
    d = (got - ref).abs().max().item()
    report["clip_text"] = dict(max_abs=d, ref_abs_max=ref.abs().max().item(), rms=(got - ref).pow(2).mean().sqrt().item())
    print(f"\nCLIP text encoder: max|d| {d:.3e} on max|h| {ref.abs().max().item():.2f}")
    assert d < 1.7e-2  # measured 8.5e-3 on max|h| 4.55 (fp16 residual stream through 12 layers)
    # causality: changing a later token must not change earlier positions
    ids2 = ids.clone()
    ids2[1, 40] = 1234
    got2 = ClipTextEngine(m)(ids2)[0]
    assert torch.equal(got2[1, :40], got[1, :40]) and not torch.equal(got2[1, 40:], got[1, 40:])


def test_pipeline_uses_the_engine_for_clip_modules(report):
    from _helpers import build_product
    from transformers import CLIPTokenizer  # noqa: F401  (presence only)
    pipe = build_product("mini", dict(lora=160))
    m = _model(1)
    pipe.text_encoder = m

    class Tok:  # ids straight through: 77 positions, BOS first
        model_max_length = 77

        def __call__(self, prompt, padding=None, max_length=77, truncation=True, return_tensors="pt"):
            n = 1 if isinstance(prompt, str) else len(prompt)
            g = torch.Generator().manual_seed(len(str(prompt)))
            ids = torch.randint(0, 49408, (n, 77), generator=g)
            return type("O", (), {"input_ids": ids, "attention_mask": torch.ones_like(ids)})()
    pipe.tokenizer = Tok()
    emb = pipe._encode_prompt("a silver jeep", pipe.unet.device, 1, True, None)
    assert emb.shape == (2, 77, 768) and pipe._clip_engine[1] is not None
    ref = torch.cat([m(pipe.tokenizer([""]).input_ids.cuda())[0], m(pipe.tokenizer("a silver jeep").input_ids.cuda())[0]])
    d = (emb - ref).abs().max().item()
    report["clip_in_pipeline"] = dict(max_abs=d)
    assert d < 2e-2 * max(1.0, ref.abs().max().item())
