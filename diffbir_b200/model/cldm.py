"""ControlLDM — drop-in counterpart of the reference's diffbir.model.ControlLDM
(model/cldm.py:20-210): same constructor arguments (the YAML `params` of
configs/inference/cldm.yaml), same checkpoint loaders, same methods and the mutable
`control_scales` list the pipeline sets per call — backed by the sm_90a kernel engines
instead of nn.Modules.  There is no eager / CPU path: every method needs the CUDA library.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Set, Tuple

import torch

from .. import arch
from ..engine.cldm import CldmEngine
from ..engine.vae import VaeEngine
from .clip import BpeTokenizer, SyntheticTokenizer, TextTower, find_bpe_vocab


def _plain(cfg) -> dict:
    out = {}
    for k, v in dict(cfg).items():
        out[k] = tuple(v) if isinstance(v, (list, tuple)) or type(v).__name__ == "ListConfig" else v
    return out


class ControlLDM:
    def __init__(self, unet_cfg, vae_cfg, clip_cfg, controlnet_cfg, latent_scale_factor,
                 device="cuda", synthetic_tokenizer: bool = False):
        self.unet_cfg = _plain(unet_cfg)
        self.controlnet_cfg = _plain(controlnet_cfg)
        dd = dict(vae_cfg["ddconfig"])
        self.vae_cfg = dict(embed_dim=vae_cfg["embed_dim"], z_channels=dd["z_channels"],
                            in_channels=dd["in_channels"], out_ch=dd["out_ch"], ch=dd["ch"],
                            ch_mult=tuple(dd["ch_mult"]), num_res_blocks=dd["num_res_blocks"])
        self.clip_cfg = dict(clip_cfg)
        self.scale_factor = latent_scale_factor
        self.control_scales = [1.0] * 13
        self.device = torch.device(device)
        self.synthetic_tokenizer = synthetic_tokenizer
        self._unet_sd = self._vae_sd = self._clip_sd = self._cn_sd = None
        self.engine: Optional[CldmEngine] = None
        self.vae: Optional[VaeEngine] = None
        self.clip: Optional[TextTower] = None
        self._tokenizer = None
        self._ctx_ref = None      # (tensor, version) the engine's cross-attention K/V were built from
        self._t_key = None
        self._txt_cache: Dict[str, torch.Tensor] = {}   # prompt -> [77, D] text-tower output (see encode_text)
        # True: VAE encode / decode are sharded over the torch.distributed ranks, by image rows un-tiled and by tiles
        # tiled (all ranks must pass the same tensors; set by the pipeline while ranks cooperate on one job: tiled /
        # batch-sharded sampling)
        self.shard_vae = False
        # False: while shard_vae is set, an un-tiled VAE stays replicated instead of row-sharded; the row-sharded one
        # agrees with one GPU only to the fp16 noise floor, the tile-sharded one bit for bit
        self.shard_vae_rows = True
        self._svae = None
        self._tvae = None

    # --------------------------------------------------------------- checkpoint loaders
    @torch.no_grad()
    def load_pretrained_sd(self, sd: Dict[str, torch.Tensor]) -> Tuple[Set[str], Set[str]]:
        """Splits an SD checkpoint by the prefixes of cldm.py:37-41; returns (unused, missing)."""
        prefixes = {"unet": "model.diffusion_model.", "vae": "first_stage_model.",
                    "clip": "cond_stage_model."}
        expected = {
            "unet": list(arch.unet_shapes(self.unet_cfg)),
            "vae": list(arch.vae_shapes(self.vae_cfg)),
            "clip": ["model." + k for k in arch.clip_text_shapes(dict(arch.CLIP_TEXT_CFG, **{
                k: v for k, v in self.clip_cfg.get("text_cfg", {}).items() if k in arch.CLIP_TEXT_CFG}))],
        }
        used, missing, parts = set(), set(), {}
        for name, pre in prefixes.items():
            part = {}
            for key in expected[name]:
                full = pre + key
                if full in sd:
                    part[key] = sd[full]
                    used.add(full)
                else:
                    missing.add(full)
            parts[name] = part
        self._unet_sd, self._vae_sd = parts["unet"], parts["vae"]
        self._clip_sd = {k[len("model."):]: v for k, v in parts["clip"].items()}
        self._invalidate()
        return set(sd.keys()) - used, missing

    @torch.no_grad()
    def load_controlnet_from_ckpt(self, sd: Dict[str, torch.Tensor]) -> None:
        exp = arch.unet_shapes(self.controlnet_cfg, True)
        extra, lack = set(sd) - set(exp), set(exp) - set(sd)
        if extra or lack:   # strict, like cldm.py:64-66
            raise RuntimeError(f"controlnet state_dict mismatch: missing {sorted(lack)[:3]}, unexpected {sorted(extra)[:3]}")
        self._cn_sd = dict(sd)
        self._invalidate()

    def _invalidate(self):
        self.engine = self.vae = self.clip = None
        self._ctx_ref = self._t_key = None
        self._txt_cache = {}
        self._svae = self._tvae = None

    def release_engine_buffers(self) -> None:
        """Frees the UNet / ControlNet engine's batch-sized buffers and graphs (see CldmEngine.release_buffers)."""
        if self.engine is not None:
            self.engine.release_buffers()
        self._ctx_ref = self._t_key = None

    def release_vae_buffers(self) -> None:
        """Frees the VAE engine's workspace and graphs (see VaeEngine.release_buffers), tiled VAE included."""
        if self.vae is not None:
            self.vae.release_buffers()
        if self._tvae is not None:
            self._tvae.release_buffers()

    def _build(self):
        if self.engine is None:
            if self._unet_sd is None or self._cn_sd is None:
                raise RuntimeError("load_pretrained_sd() and load_controlnet_from_ckpt() must be called first")
            self.engine = CldmEngine(self._unet_sd, self._cn_sd, self.unet_cfg, self.controlnet_cfg, self.device)
        if self.vae is None:
            self.vae = VaeEngine(self._vae_sd, self.vae_cfg, self.device)
        if self.clip is None and self._clip_sd:
            tc = self.clip_cfg.get("text_cfg", {})
            self.clip = TextTower(self._clip_sd, heads=tc.get("heads", 16),
                                  layer=self.clip_cfg.get("layer", "penultimate"), device=self.device)

    # nn.Module-flavoured no-ops so reference-style loader code keeps working
    def eval(self):
        return self

    def to(self, device):
        if torch.device(device) != self.device:
            self.device = torch.device(device)
            self._invalidate()
        return self

    def cast_dtype(self, dtype: torch.dtype) -> "ControlLDM":
        """Kept for API compatibility (cldm.py:174-210). Precision is fixed by the kernels: 16-bit
        tensor-core operands, fp32 accumulation, fp32 residual stream and normalisation."""
        return self

    # --------------------------------------------------------------- conditioning
    def tokenize(self, txt: List[str]) -> torch.Tensor:
        if self._tokenizer is None:
            path = find_bpe_vocab()
            if path is not None:
                self._tokenizer = BpeTokenizer(path)
            elif self.synthetic_tokenizer:
                self._tokenizer = SyntheticTokenizer(self._clip_sd["token_embedding.weight"].shape[0])
            else:
                raise FileNotFoundError(
                    "CLIP BPE vocabulary not found: set DIFFBIR_BPE_VOCAB to bpe_simple_vocab_16e6.txt.gz "
                    "(or construct ControlLDM(synthetic_tokenizer=True) for synthetic checkpoints)")
        return self._tokenizer(txt)

    TXT_CACHE_MAX = 64

    @torch.no_grad()
    def encode_text(self, txt: List[str]) -> torch.Tensor:
        """FrozenOpenCLIPEmbedder.forward (model/clip.py:56-61) -> fp32 [len(txt), 77, D]. The output is a
        pure function of the prompt string and the frozen weights, so it is kept per prompt: a folder of
        images restored with the same positive / negative prompt (the CLI default) runs the text tower
        once instead of twice per image. Distinct new prompts of one call share one batched tower pass."""
        self._build()
        new = [t for t in dict.fromkeys(txt) if t not in self._txt_cache]
        if new:
            emb = self.clip(self.tokenize(new))
            if len(self._txt_cache) + len(new) > self.TXT_CACHE_MAX:
                self._txt_cache.clear()
            for t, e in zip(new, emb):
                self._txt_cache[t] = e.clone()
        return torch.stack([self._txt_cache[t] for t in txt], 0)

    @torch.no_grad()
    def vae_encode(self, image: torch.Tensor, sample: bool = True, tiled: bool = False,
                   tile_size: int = -1) -> torch.Tensor:
        """tiled: the reference's Tiled-VAE semantics (engine.vae_tiled), tile_size in image pixels."""
        self._build()
        image = image.to(self.device, torch.float32).contiguous()
        if tiled:
            m = self.tiled_vae().encode_moments(image, tile_size)
        else:
            sv = self._sharded_vae(image.shape[2], image.shape[3])
            m = sv.encode_moments(image) if sv is not None else self.vae.encode_moments(image)
        mean, logvar = m.chunk(2, dim=1)
        if sample:   # DiagonalGaussianDistribution.sample, model/distributions.py:25-37
            std = torch.exp(0.5 * torch.clamp(logvar, -30.0, 20.0))
            mean = mean + std * torch.randn(mean.shape).to(self.device)
        return mean * self.scale_factor

    @torch.no_grad()
    def vae_decode(self, z: torch.Tensor, tiled: bool = False, tile_size: int = -1) -> torch.Tensor:
        """tiled: the reference's Tiled-VAE semantics (engine.vae_tiled), tile_size in latent pixels."""
        self._build()
        z = (z / self.scale_factor).to(self.device, torch.float32).contiguous()
        if tiled:
            return self.tiled_vae().decode(z, tile_size)
        sv = self._sharded_vae(8 * z.shape[2], 8 * z.shape[3])
        return sv.decode(z) if sv is not None else self.vae.decode(z)

    def tiled_vae(self):
        """The tiled VAE (engine.vae_tiled) on this model's VAE weights. While shard_vae is set and more than one
        rank cooperates, each rank runs its share of the tiles and every rank returns the full result (the
        row-sharded VAE computes the un-tiled semantics, so it is not used here); otherwise it runs by itself."""
        self._build()
        import torch.distributed as dist
        world = dist.get_world_size() if self.shard_vae and dist.is_available() and dist.is_initialized() else 1
        if self._tvae is None or self._tvae.world != world:
            from ..engine.vae_tiled import TiledVae
            self._tvae = TiledVae(self.vae, dist.get_rank() if world > 1 else 0, world)
        return self._tvae

    def _sharded_vae(self, h_img: int, w_img: int):
        """The row-sharded VAE (engine.vae_sharded) when ranks cooperate on this job and the size allows it."""
        if not (self.shard_vae and self.shard_vae_rows):
            return None
        from ..engine.vae_sharded import ShardedVae
        if not ShardedVae.usable(h_img, w_img):
            return None
        if self._svae is None:
            self._svae = ShardedVae(self.vae)
        return self._svae

    @torch.no_grad()
    def prepare_condition(self, cond_img: torch.Tensor, txt: List[str], tiled: bool = False,
                          tile_size: int = -1) -> Dict[str, torch.Tensor]:
        self._build()
        return dict(c_txt=self.encode_text(list(txt)),
                    c_img=self.vae_encode(cond_img * 2 - 1, sample=False, tiled=tiled, tile_size=tile_size))

    @torch.no_grad()
    def prepare_condition_pair(self, cond_img: torch.Tensor, pos_txt: List[str], neg_txt: List[str],
                               tiled: bool = False, tile_size: int = -1):
        """(cond, uncond) of Pipeline.apply_cldm (pipeline.py:116-128): the condition image is encoded
        once (the posterior mode is deterministic, the reference encodes the same image twice) and both
        prompt lists share one batched text-tower call."""
        self._build()
        n = len(pos_txt)
        c_txt = self.encode_text(list(pos_txt) + list(neg_txt))
        c_img = self.vae_encode(cond_img * 2 - 1, sample=False, tiled=tiled, tile_size=tile_size)
        return (dict(c_txt=c_txt[:n].contiguous(), c_img=c_img),
                dict(c_txt=c_txt[n:].contiguous(), c_img=c_img.clone()))

    @torch.no_grad()
    def prepare_condition_pairs(self, cond_img: torch.Tensor, pos_txt: List[str], neg_txt: str,
                                tiled: bool = False, tile_size: int = -1):
        """prepare_condition_pair with a positive prompt per image. Image i's text rows are what Pipeline.run of that
        image alone computes on an empty cache: (pos_txt[i], neg_txt) as one text-tower batch of 2. The tower's
        rows depend on its batch size, so they are neither read from nor written to the per-prompt cache, whose
        entries may come from batches of another size. A distinct positive prompt is encoded once per call."""
        self._build()
        pairs = {p: self.clip(self.tokenize([p, neg_txt])) for p in dict.fromkeys(pos_txt)}
        c_img = self.vae_encode(cond_img * 2 - 1, sample=False, tiled=tiled, tile_size=tile_size)
        return (dict(c_txt=torch.stack([pairs[p][0] for p in pos_txt]), c_img=c_img),
                dict(c_txt=torch.stack([pairs[p][1] for p in pos_txt]), c_img=c_img.clone()))

    # --------------------------------------------------------------- denoiser
    @torch.no_grad()
    def forward(self, x_noisy: torch.Tensor, t: torch.Tensor, cond: Dict[str, torch.Tensor]) -> torch.Tensor:
        """Generic entry (any sampler can call it): cldm.py:160-172. Context K/V and the time
        embedding are cached on the identity (+ in-place version) of c_txt / the value of t."""
        self._build()
        eng = self.engine
        nb = x_noisy.shape[0]
        tv = t.reshape(-1)
        t0 = int(tv[0].item())
        if nb > 1 and not bool((tv == tv[0]).all()):
            raise NotImplementedError("per-sample timesteps in one batch are not used by the samplers")
        c_txt = cond["c_txt"]
        # identity + version of a tensor we keep alive: a freed prompt's address can be handed to the
        # next prompt by the caching allocator, so (data_ptr, shape) alone is not a safe key
        ref = self._ctx_ref
        if ref is None or ref[0] is not c_txt or ref[1] != c_txt._version:
            eng.set_context(c_txt.to(self.device, torch.float32))
            self._ctx_ref = (c_txt, c_txt._version)
        if (t0, nb) != self._t_key:
            eng.set_timesteps([t0], nb)
            eng.load_step(0)
            self._t_key = (t0, nb)
        return eng.forward(x_noisy.to(self.device, torch.float32).contiguous(),
                           cond["c_img"].to(self.device, torch.float32).contiguous(), self.control_scales)

    __call__ = forward
