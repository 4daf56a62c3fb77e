"""Fixture for the RAM++ captioner, produced by the REFERENCE module RAM_plus(image_size=384, vit="swin_l")
(ram/models/ram_plus.py) on the CPU in fp32 with seeded synthetic weights loaded into it (which also pins
diffbir_b200.arch.ram_shapes):

    python tests/golden/gen_golden_ram.py          # needs /root/reference; writes ram_small.npz (no network)

Synthetic weights give logits of a few tenths around zero, so almost every class would sit next to its threshold.
The generator therefore rescales `fc` (weight x fc_scale, bias = fc_bias, both stored) so that between 5 and 50
tags fire and no class's probability lies within 0.01 of its threshold; it walks the seed until both hold. The
fixture stores seeds, the two fc numbers, the reference's 4585 class thresholds, the rebuilt input's checksum,
every 64th row of each stage's output, image_embeds, the logits, the decisions and the caption.
"""
import os
import sys
from pathlib import Path

os.environ["HF_HUB_OFFLINE"] = "1"
os.environ["TRANSFORMERS_OFFLINE"] = "1"

import numpy as np  # noqa: E402
import torch  # noqa: E402
# before the oracle's shims join sys.path: their accelerate stand-in has no version for transformers to check
import transformers.modeling_utils as mu  # noqa: E402
import transformers.pytorch_utils as pu  # noqa: E402

sys.path.insert(0, str(Path(__file__).resolve().parent))
from _ref_import import REFERENCE, use_reference  # noqa: E402

use_reference()
sys.path.insert(0, str(REFERENCE))
from diffbir_b200 import arch  # noqa: E402
from diffbir_b200.utils.synth import make_state_dict  # noqa: E402
from oracle import ram as oram  # noqa: E402

OUT = Path(__file__).resolve().parent
IMAGE_SEED = 384
STAGE_ROW_STEP = 64


def fixture_image(seed: int = IMAGE_SEED) -> torch.Tensor:
    """The ToTensor() image in [0, 1], [1, 3, 384, 384] (the rebuilt input)."""
    return torch.rand(1, 3, 384, 384, generator=torch.Generator().manual_seed(seed))


def reference_model():
    """RAM_plus with the import-time workarounds the reference needs on transformers 5.5 without network."""
    for n in ("apply_chunking_to_forward", "prune_linear_layer"):
        setattr(mu, n, getattr(pu, n))
    mu.find_pruneable_heads_and_indices = None               # only used by prune_heads
    mu.PreTrainedModel.init_weights = lambda self: None       # the weights are replaced anyway
    mu.PreTrainedModel.resize_token_embeddings = lambda self, *a, **k: None
    mu.PreTrainedModel.get_head_mask = lambda self, head_mask, n, *a, **k: [None] * n

    def invert_attention_mask(self, m):
        e = (m[:, None, None, :] if m.dim() == 2 else m[:, None, :, :]).to(torch.float32)
        return (1.0 - e) * torch.finfo(torch.float32).min
    mu.PreTrainedModel.invert_attention_mask = invert_attention_mask
    import ram.models.ram_plus  # noqa: F401  (the package's ram_plus function shadows the module name)
    rp = sys.modules["ram.models.ram_plus"]

    class Tokenizer:                                          # BertTokenizer.from_pretrained would download
        def __len__(self):
            return 30524
    rp.init_tokenizer = lambda *a, **k: Tokenizer()
    return rp.RAM_plus(image_size=384, vit="swin_l").eval()


def synthetic_sd(seed: int, fc_scale: float = 1.0, fc_bias: float = 0.0):
    sd = make_state_dict(arch.ram_shapes(arch.RAM_CFG), seed)
    sd["fc.weight"] = sd["fc.weight"] * fc_scale
    sd["fc.bias"] = torch.full((1,), fc_bias)
    return sd


@torch.no_grad()
def main():
    model = reference_model()
    thr = model.class_threshold.clone()
    tags = list(model.tag_list)
    x01 = fixture_image()
    x = oram.normalize(x01)
    for seed in range(11, 40):
        sd = synthetic_sd(seed)
        missing, unexpected = model.load_state_dict(sd, strict=False)
        assert not unexpected and all("relative_position_index" in k or "attn_mask" in k for k in missing), missing
        # the fc input is fixed by the other weights: rescale fc from the reference's logits at scale 1, bias 0
        feats, stages = {}, []
        h = model.fc.register_forward_hook(lambda m, i_, o: feats.update(inp=i_[0].clone()))
        model.generate_tag(x)
        h.remove()
        base = feats["inp"][0] @ sd["fc.weight"][0]                 # [classes], bias 0
        fc_scale = float(30.0 / base.std())
        logit_thr = torch.log(thr / (1 - thr))
        # bias so that about 20 classes fire: the 20th largest of (scaled logit - threshold logit)
        fc_bias = float(-(base * fc_scale - logit_thr).sort(descending=True).values[20:22].mean())
        sd = synthetic_sd(seed, fc_scale, fc_bias)
        model.load_state_dict(sd, strict=False)
        hooks = [model.visual_encoder.layers[i].blocks[-1].register_forward_hook(
            lambda m, i_, o: stages.append(o.clone())) for i in range(4)]
        feats.clear()
        hk2 = model.image_proj.register_forward_hook(lambda m, i_, o: feats.update(emb=o.clone()))
        h = model.fc.register_forward_hook(lambda m, i_, o: feats.update(logits=o.clone()))
        tag_out, _ = model.generate_tag(x)
        for hk in hooks + [hk2, h]:
            hk.remove()
        logits = feats["logits"][0, :, 0]
        prob = torch.sigmoid(logits)
        fired = (prob > thr).nonzero().flatten().tolist()
        margin = float((prob - thr).abs().min())
        print(f"seed {seed}: {len(fired)} tags, smallest margin {margin:.4f}")
        if 5 <= len(fired) <= 50 and margin > 0.01:
            break
    else:
        raise SystemExit("no seed met the tag-count and margin conditions")
    caption = tag_out[0].replace(" | ", ", ")
    assert caption == ", ".join(tags[i] for i in fired)
    np.savez_compressed(
        OUT / "ram_small.npz", seed=seed, image_seed=IMAGE_SEED, fc_scale=np.float64(fc_scale),
        fc_bias=np.float64(fc_bias), x_sum=np.float64(x01.double().sum()), thresholds=thr.numpy(),
        stage_row_step=STAGE_ROW_STEP, **{f"stage{i}": s[0, ::STAGE_ROW_STEP].numpy() for i, s in enumerate(stages)},
        image_embeds=feats["emb"][0].numpy(), logits=logits.numpy(), decisions=(prob > thr).numpy(),
        fired=np.array(fired, dtype=np.int32), fired_tags=np.array([tags[i] for i in fired]), caption=np.array(caption),
        min_margin=np.float64(margin))
    print(f"wrote ram_small.npz: seed {seed}, {len(fired)} tags, margin {margin:.4f}: {caption}")


if __name__ == "__main__":
    main()
