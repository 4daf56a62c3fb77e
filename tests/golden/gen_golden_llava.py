"""Fixture for the LLaVA captioner, produced by the REFERENCE modules (llava/model/language_model/llava_llama.py,
llava/mm_utils.py) on the CPU in fp32 at a reduced size, with seeded synthetic weights loaded into them (which also
pins diffbir_b200.arch.llava_shapes):

    python tests/golden/gen_golden_llava.py        # needs /root/reference; writes llava_small.npz (no network)

- LlavaLlamaForCausalLM at hidden 256, 2 layers, 2 heads x 128, SwiGLU 512, vocab 512. Its vision tower is a
  CLIPVisionTower whose CLIPVisionModel (3 layers, 2 heads x 64, MLP 256, the real 336 / 14 geometry, 576 patches)
  is assigned directly, so from_pretrained never runs.
- The prompt ids come from the reference's tokenizer_image_token over the llava_v1 prompt, with a byte tokenizer in
  LLaMA's byte-fallback layout (ids 3 .. 258 = bytes, BOS 1) standing in for the SentencePiece model.
- The pixel values come from the reference's process_images (image_aspect_ratio "pad") with transformers' PIL
  CLIPImageProcessor constructed locally with the openai/clip-vit-large-patch14-336 settings, for a non-square
  200 x 300 image.
- Greedy tokens come from the reference's own generate when it runs under the installed transformers; otherwise the
  generator drives the reference model's forward with its past_key_values in a greedy loop (same computation: argmax
  of the last position's logits, one token per step). `greedy_source` records which.
- lm_head is scaled by lm_head_scale (stored) and the seed is walked until none of the 16 tokens is EOS, they hold
  at least 3 distinct ids (random weights tend to repeat one token) and every step's top-1 logit margin is at least
  0.05 (stored as min_margin).

Stored: seeds, the scale, the config, the ids, every 8th row of the pixel values and their sum, every 4th row of the
image features and their sum, the prefill logits, the 16 tokens and the teacher-forced logits of those steps.
"""
import json
import os
import sys
import types
from pathlib import Path

os.environ["HF_HUB_OFFLINE"] = "1"
os.environ["TRANSFORMERS_OFFLINE"] = "1"

import numpy as np  # noqa: E402
import torch  # noqa: E402
import transformers.modeling_utils as mu  # noqa: E402,F401
from PIL import Image  # noqa: E402

sys.path.insert(0, str(Path(__file__).resolve().parent))
from _ref_import import REFERENCE, use_reference  # noqa: E402

use_reference()
sys.path.insert(0, str(REFERENCE))
from diffbir_b200 import arch  # noqa: E402
from diffbir_b200.utils.synth import make_state_dict, synthetic_lq  # noqa: E402

OUT = Path(__file__).resolve().parent
CFG = dict(arch.LLAVA_CFG, vocab=512, hidden=256, layers=2, heads=2, intermediate=512, v_width=128, v_layers=3,
           v_heads=2, v_intermediate=256)
IMAGE_SEED = 7
LM_HEAD_SCALE = 4.0
STEPS = 16
PIXEL_ROW_STEP = 8
FEATURE_ROW_STEP = 4
PROMPT = ("A chat between a curious human and an artificial intelligence assistant. The assistant gives helpful, "
          "detailed, and polite answers to the human's questions. USER: <image>\n"
          "Please give me a very short description of this image. ASSISTANT:")


class ByteTokenizer:
    bos_token_id = 1

    def __call__(self, text):
        return types.SimpleNamespace(input_ids=[1] + [3 + b for b in text.encode("utf-8")])


def fixture_sd(seed: int):
    sd = make_state_dict(arch.llava_shapes(CFG), seed)
    sd["lm_head.weight"] = sd["lm_head.weight"] * LM_HEAD_SCALE
    return sd


def build_model(sd):
    from transformers import CLIPVisionConfig, CLIPVisionModel
    from llava.model.language_model.llava_llama import LlavaConfig, LlavaLlamaForCausalLM
    from llava.model.multimodal_encoder.clip_encoder import CLIPVisionTower
    from llava.model.multimodal_projector.builder import build_vision_projector
    config = LlavaConfig(vocab_size=CFG["vocab"], hidden_size=CFG["hidden"], intermediate_size=CFG["intermediate"],
                         num_hidden_layers=CFG["layers"], num_attention_heads=CFG["heads"],
                         num_key_value_heads=CFG["heads"], rms_norm_eps=CFG["rms_eps"], rope_theta=CFG["rope_theta"],
                         max_position_embeddings=2048, bos_token_id=1, eos_token_id=2, pad_token_id=0,
                         tie_word_embeddings=False, attn_implementation="eager")
    config.mm_projector_type = "mlp2x_gelu"
    config.mm_hidden_size = CFG["v_width"]
    config.mm_vision_select_layer = CFG["select_layer"]
    config.mm_vision_select_feature = "patch"
    config.image_aspect_ratio = "pad"
    config.mm_use_im_start_end = False
    model = LlavaLlamaForCausalLM(config)
    tower = CLIPVisionTower.__new__(CLIPVisionTower)
    torch.nn.Module.__init__(tower)
    tower.is_loaded = True
    tower.vision_tower_name = "openai/clip-vit-large-patch14-336"
    tower.select_layer = CFG["select_layer"]
    tower.select_feature = "patch"
    tower.vision_tower = CLIPVisionModel(CLIPVisionConfig(
        hidden_size=CFG["v_width"], intermediate_size=CFG["v_intermediate"], num_hidden_layers=CFG["v_layers"],
        num_attention_heads=CFG["v_heads"], image_size=CFG["image"], patch_size=CFG["patch"],
        layer_norm_eps=CFG["v_eps"], hidden_act="quick_gelu", attn_implementation="eager"))
    model.model.vision_tower = tower
    model.model.mm_projector = build_vision_projector(config)
    missing, unexpected = model.load_state_dict(sd, strict=False)
    missing = [k for k in missing if not k.endswith(("position_ids", "inv_freq"))]
    assert not missing and not unexpected, (missing[:4], unexpected[:4])
    return model.float().eval()


def image_processor():
    from transformers.models.clip.image_processing_pil_clip import CLIPImageProcessorPil
    return CLIPImageProcessorPil(size={"shortest_edge": 336}, crop_size={"height": 336, "width": 336},
                                 do_center_crop=True, image_mean=[0.48145466, 0.4578275, 0.40821073],
                                 image_std=[0.26862954, 0.26130258, 0.27577711], resample=3)


def greedy_by_forward(model, ids, pixel_values, steps):
    out = model(input_ids=ids, images=pixel_values, use_cache=True)
    past, toks = out.past_key_values, []
    logits = out.logits[0, -1]
    for _ in range(steps):
        t = int(logits.argmax())
        toks.append(t)
        out = model(input_ids=torch.tensor([[t]]), past_key_values=past, use_cache=True)
        past, logits = out.past_key_values, out.logits[0, -1]
    return toks


@torch.no_grad()
def run(seed: int):
    from llava.mm_utils import process_images, tokenizer_image_token
    model = build_model(fixture_sd(seed))
    ids = tokenizer_image_token(PROMPT, ByteTokenizer(), -200)
    img = Image.fromarray(synthetic_lq(200, 300, seed=IMAGE_SEED)[0])
    pixel_values = process_images([img], image_processor(), model.config)
    input_ids = torch.tensor([ids])
    feats = model.encode_images(pixel_values)[0]
    source = "generate"
    try:
        gen = model.generate(input_ids, images=pixel_values, image_sizes=[img.size], do_sample=False, num_beams=1,
                             max_new_tokens=STEPS, use_cache=True)
        toks = gen[0].tolist()             # inputs_embeds generation: only the new tokens come back
        if len(toks) < STEPS:              # stopped at EOS: this seed is walked past
            return None
    except Exception as e:                                                # noqa: BLE001
        print(f"generate does not run under this transformers ({type(e).__name__}: {e}); greedy loop over forward")
        source = "forward"
        toks = greedy_by_forward(model, input_ids, pixel_values, STEPS)
    # teacher-forced logits: the prompt, then the tokens one at a time
    out = model(input_ids=input_ids, images=pixel_values, use_cache=True)
    rows, past = [out.logits[0, -1]], out.past_key_values
    for t in toks[:-1]:
        out = model(input_ids=torch.tensor([[t]]), past_key_values=past, use_cache=True)
        rows.append(out.logits[0, -1])
        past = out.past_key_values
    forced = torch.stack(rows)
    assert [int(r.argmax()) for r in forced] == toks
    top2 = forced.topk(2, -1).values
    margin = float((top2[:, 0] - top2[:, 1]).min())
    return dict(ids=np.array(ids, np.int64), pixel_values=pixel_values[0].numpy(), feats=feats.numpy(),
                tokens=np.array(toks, np.int64), forced=forced.numpy(), margin=margin, source=source)


def main():
    for seed in range(100, 200):
        r = run(seed)
        if r is None:
            continue
        print(f"seed {seed}: tokens {r['tokens'].tolist()} margin {r['margin']:.4f}")
        if 2 not in r["tokens"].tolist() and len(set(r["tokens"].tolist())) >= 3 and r["margin"] >= 0.05:
            break
    else:
        raise SystemExit("no seed met the margin")
    pv, feats = r["pixel_values"], r["feats"]
    np.savez_compressed(
        OUT / "llava_small.npz", seed=seed, image_seed=IMAGE_SEED, lm_head_scale=LM_HEAD_SCALE, cfg=json.dumps(CFG),
        input_ids=r["ids"], pixel_rows=pv[:, ::PIXEL_ROW_STEP], pixel_row_step=PIXEL_ROW_STEP,
        pixel_sum=float(np.float64(pv).sum()), feature_rows=feats[::FEATURE_ROW_STEP],
        feature_row_step=FEATURE_ROW_STEP, feature_sum=float(np.float64(feats).sum()), prefill_logits=r["forced"][0],
        tokens=r["tokens"], forced_logits=r["forced"], min_margin=r["margin"], greedy_source=r["source"])
    print("wrote", OUT / "llava_small.npz", "greedy from", r["source"])


if __name__ == "__main__":
    main()
