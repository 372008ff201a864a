"""`LatentDiffusion` / `create_latent_diffusion`: the reference's training wrapper surface
(micro_diffusion/models/model.py) over the CUDA engine.

`forward(batch)` returns `(loss, latents, conditioning)` exactly like the reference (model.py:104-142); the
loss tensor carries a single autograd node whose backward runs the hand-written CUDA backward and writes
parameter gradients straight into the flat gradient buffer behind `p.grad` (see models/dit.py).
Random draws keep the reference's order and generators -- torch.randn([B,1,1,1]) -> self.randn_like(x) ->
torch.rand(B,T) (model.py:182,188; utils.py:390) -- so a seeded run consumes the RNG stream identically.
"""
from __future__ import annotations

from functools import partial
from typing import Optional

import numpy as np
import torch
import torch.nn as nn

from . import dit as model_zoo
from .utils import DATA_TYPES, DistLoss, text_encoder_embedding_format

try:  # Composer is optional here; with it installed LatentDiffusion is a real ComposerModel
    from composer.models import ComposerModel as _Base
except Exception:  # pragma: no cover
    _Base = nn.Module


class _AttrDict(dict):
    __getattr__ = dict.__getitem__
    __setattr__ = dict.__setitem__


class _EDMLossFn(torch.autograd.Function):
    """loss = edm_loss(...) with the whole forward and backward executed by the engine."""

    @staticmethod
    def forward(ctx, anchor, ld, lat, cap, drop, rnd, eps_noise, mask_ratio, mask_noise, cap_out, keep):
        eng = ld.dit.engine
        # `keep` = grad mode at the call site (inside Function.forward torch.is_grad_enabled() is always False and
        # ctx.needs_input_grad ignores no_grad).  Under no_grad (eval_forward / Trainer.evaluate) nothing is saved,
        # like the reference's no_grad evaluation.
        keep = bool(keep and ctx.needs_input_grad[0])
        c = eng.forward_loss(lat, cap, drop, rnd, eps_noise, mask_ratio, mask_noise, ld._edm_scalars(), keep=keep,
                             cap_out=cap_out)
        ctx.ld, ctx.c = ld, (c if keep else None)
        ld.last_per_sample_loss = c.per_sample
        return c.loss.reshape(())

    @staticmethod
    def backward(ctx, gout):
        ld, c = ctx.ld, ctx.c
        if c is None:
            raise RuntimeError("MicroDiT loss: no saved activations (backward called twice, or the forward ran without "
                               "a gradient-requiring anchor)")
        ld.dit.prepare_grads()
        gscale = gout.detach().reshape(1).to(torch.float32).contiguous()
        ld.dit.engine.backward(c, gscale)
        ctx.c = None  # free the saved activations
        return (None,) * 11


class LatentDiffusion(_Base):
    def __init__(self, dit: nn.Module, vae, text_encoder, tokenizer, image_key: str = "image", text_key: str = "captions",
                 image_latents_key: str = "image_latents", text_latents_key: str = "caption_latents",
                 precomputed_latents: bool = True, dtype: str = "bfloat16", latent_res: int = 32, p_mean: float = -0.6,
                 p_std: float = 1.2, train_mask_ratio: float = 0.0):
        super().__init__()
        self.dit = dit
        self.vae = vae
        self.image_key, self.text_key = image_key, text_key
        self.image_latents_key, self.text_latents_key = image_latents_key, text_latents_key
        self.precomputed_latents = precomputed_latents
        self.dtype = dtype
        self.latent_res = latent_res
        self.edm_config = _AttrDict(sigma_min=0.002, sigma_max=80, P_mean=p_mean, P_std=p_std, sigma_data=0.9,
                                    num_steps=18, rho=7, S_churn=0, S_min=0, S_max=float("inf"), S_noise=1)
        self.train_mask_ratio = train_mask_ratio
        self.eval_mask_ratio = 0.0
        assert self.train_mask_ratio >= 0, "Masking ratio must be non-negative!"
        self.randn_like = torch.randn_like
        self.latent_scale = self.vae.config.scaling_factor
        self.text_encoder = text_encoder
        self.tokenizer = tokenizer
        self.text_encoder.requires_grad_(False)
        self.vae.requires_grad_(False)
        try:  # FSDP wrap hints read by Composer (model.py:100-102)
            self.text_encoder._fsdp_wrap = False
            self.vae._fsdp_wrap = False
        except Exception:
            pass
        self.dit._fsdp_wrap = True
        self.last_per_sample_loss = None
        self.cache_prompt = True  # sampler fast path: caption-only work once per edm_sampler_loop (engine.prompt_cache)
        self._prompt_memo = None
        # sampler fast path: the Heun loop as replays of captured CUDA graphs where _sampler_graph_eligible holds; False
        # keeps the eager loop (A/B runs, and the comparator of the graph path's tests)
        self.sampler_graph = True
        self.sampler_debug = None  # optional callable(step, call, D): sees the fp32 denoiser output of every sampler call

    def _edm_scalars(self):
        e = self.edm_config
        return {"P_mean": float(e.P_mean), "P_std": float(e.P_std), "sigma_data": float(e.sigma_data)}

    # ------------------------------------------------------------------ training forward (model.py:104-142)
    def forward(self, batch: dict):
        if self.precomputed_latents and self.image_latents_key in batch:
            latents = batch[self.image_latents_key]
        else:
            with torch.no_grad():
                images = batch[self.image_key]
                latents = self.vae.encode(images.to(DATA_TYPES[self.dtype]))["latent_dist"].sample().data
                latents *= self.latent_scale
        if self.precomputed_latents and self.text_latents_key in batch:
            conditioning = batch[self.text_latents_key]
        else:
            captions = batch[self.text_key]
            captions = captions.view(-1, captions.shape[-1])
            if "attention_mask" in batch:
                conditioning = self.text_encoder.encode(
                    captions, attention_mask=batch["attention_mask"].view(-1, captions.shape[-1]))[0]
            else:
                conditioning = self.text_encoder.encode(captions)[0]
        drop = batch["drop_caption_mask"] if "drop_caption_mask" in batch.keys() else None
        loss = self._edm_loss_impl(latents, conditioning, drop,
                                   self.train_mask_ratio if self.training else self.eval_mask_ratio,
                                   inplace_caption_mask=True)
        return (loss, latents, conditioning)

    def _edm_loss_impl(self, x, y, drop, mask_ratio, inplace_caption_mask=False):
        dit = self.dit
        dev = x.device
        if x.dtype not in (torch.float16, torch.float32):
            x = x.float()
        x = x.contiguous()
        if y.dtype != torch.float16:
            y = y.to(torch.float16)
            inplace_caption_mask = False
        y = y.contiguous()
        if drop is not None:
            drop = drop.to(device=dev, dtype=torch.float64).contiguous()
        B = x.shape[0]
        rnd_normal = torch.randn([B, 1, 1, 1], device=dev)                      # model.py:182
        eps_noise = self.randn_like(x.float() if x.dtype != torch.float32 else x)  # model.py:188 (hookable)
        mask_noise = None
        if mask_ratio > 0:
            assert dit.training, "Masking is only recommended during training"   # model.py:204-206
            mask_noise = torch.rand(B, dit.cfg.num_patches, device=dev)          # utils.py:390
        dit.engine  # bind storage / anchor before the autograd node is built
        return _EDMLossFn.apply(dit._anchor, self, x, y, drop, rnd_normal.reshape(B).contiguous(),
                                eps_noise.contiguous(), float(mask_ratio), mask_noise,
                                y if (inplace_caption_mask and drop is not None) else None, torch.is_grad_enabled())

    def edm_loss_with_draws(self, x, y, drop, rnd_normal, eps_noise, mask_noise, mask_ratio: float) -> torch.Tensor:
        """edm_loss with the three random draws supplied by the caller (seeded replay / parity tests):
        rnd_normal (B,), eps_noise like x (f32), mask_noise (B,T) uniform or None."""
        dev = self.dit.store.device
        x = x.to(dev).contiguous()
        y = y.to(device=dev, dtype=torch.float16).contiguous()
        if drop is not None:
            drop = drop.to(device=dev, dtype=torch.float64).contiguous()
        self.dit.engine
        return _EDMLossFn.apply(self.dit._anchor, self, x, y, drop, rnd_normal.to(dev).float().reshape(-1).contiguous(),
                                eps_noise.to(dev).float().contiguous(), float(mask_ratio),
                                mask_noise.to(dev).float().contiguous() if mask_noise is not None else None, None,
                                torch.is_grad_enabled())

    def edm_loss(self, x: torch.Tensor, y: torch.Tensor, mask_ratio: float = 0, **kwargs) -> torch.Tensor:
        """model.py:181-210 (x: latents, y: caption embeddings (B,1,L,Dc))."""
        return self._edm_loss_impl(x, y, None, mask_ratio)

    def model_forward_wrapper(self, x, sigma, y, model_forward_fxn, mask_ratio: float, **kwargs) -> dict:
        """EDM preconditioning around the denoiser (model.py:144-179).  The fused kernel path (no gradients) is taken
        when `model_forward_fxn` is this model's own DiT (plain or CFG partial) and no gradient is wanted; under grad
        mode with x, sigma, y or a DiT parameter requiring grad, and for any other function, the reference's own
        composition c_skip*x + c_out*F(c_in*x, ln(sigma)/4, y) runs over the (differentiable) DiT.forward."""
        own, cfg = self._own_forward(model_forward_fxn)
        B = x.shape[0]
        sigma_b = sigma.to(torch.float32).reshape(-1).expand(B).contiguous()
        fused = own and not self._wants_grad(x, sigma, y)
        if fused and not (torch.is_grad_enabled() and self.dit.training and mask_ratio > 0):
            with torch.no_grad():
                eng = self.dit.engine
                xin = x.float().contiguous()
                cap = self.dit._caption_f16(y)
                memo = self.__dict__.get("_prompt_memo")  # set by edm_sampler_loop for the duration of one run
                if memo is not None and (memo["y"] is not y or memo["cfg"] != cfg):
                    memo = None
                if cfg != 1.0:  # DiT.forward_with_cfg (dit.py:521-550) around the fused denoiser
                    xin2 = torch.cat([xin, xin], 0)
                    sg2 = torch.cat([sigma_b, sigma_b], 0)
                    if memo is not None and memo["pc"] is None:
                        memo["cap"] = torch.cat([cap, torch.zeros_like(cap)], 0)
                        memo["pc"] = eng.prompt_cache(memo["cap"])
                    cap2 = memo["cap"] if memo is not None else torch.cat([cap, torch.zeros_like(cap)], 0)
                    _, fx, _ = eng.denoise(xin2, sg2, cap2, 0.0, None, self._edm_scalars(), want_raw=True,
                                           prompt=memo["pc"] if memo is not None else None)
                    cond, unc = torch.split(fx, B, dim=0)
                    f = unc + cfg * (cond - unc)
                    sd = self.edm_config.sigma_data
                    sg = sigma_b.view(-1, 1, 1, 1)
                    d = (sd ** 2 / (sg ** 2 + sd ** 2)) * xin + (sg * sd / (sg ** 2 + sd ** 2).sqrt()) * f
                    return {"sample": d}
                noise = torch.rand(B, self.dit.cfg.num_patches, device=x.device) if mask_ratio > 0 else None
                if memo is not None and memo["pc"] is None:
                    memo["pc"] = eng.prompt_cache(cap)
                d, _, mask = eng.denoise(xin, sigma_b, cap, mask_ratio, noise, self._edm_scalars(),
                                         prompt=memo["pc"] if memo is not None else None)
                return {"sample": d, "mask": mask}
        sd = self.edm_config.sigma_data
        sg = sigma_b.to(x.dtype).reshape(-1, 1, 1, 1)
        c_skip = sd ** 2 / (sg ** 2 + sd ** 2)
        c_out = sg * sd / (sg ** 2 + sd ** 2).sqrt()
        c_in = 1 / (sd ** 2 + sg ** 2).sqrt()
        out = model_forward_fxn((c_in * x).to(x.dtype), (sg.log() / 4).flatten(), y, mask_ratio=mask_ratio, **kwargs)
        out["sample"] = c_skip * x + c_out * out["sample"]
        return out

    def _own_forward(self, fn):
        """(True, cfg) when fn is this model's own DiT -- the module, its forward, or the CFG partial of its forward --
        and (False, 1.0) for any other function."""
        cfg = 1.0
        if isinstance(fn, partial) and getattr(fn.func, "__self__", None) is self.dit:
            cfg = fn.keywords.get("cfg", 1.0)
            fn = fn.func
        return fn is self.dit or getattr(fn, "__self__", None) is self.dit, cfg

    def _wants_grad(self, x, sigma, y) -> bool:
        """Grad mode is on and a gradient is wanted for an input or for the DiT's parameters."""
        if not torch.is_grad_enabled():
            return False
        return (any(torch.is_tensor(v) and v.requires_grad for v in (x, sigma, y))
                or any(p.requires_grad for p in self.dit.parameters()))

    # ------------------------------------------------------------------ Composer hooks (model.py:213-229)
    def loss(self, outputs: tuple, batch: dict) -> torch.Tensor:
        return outputs[0]

    def eval_forward(self, batch: dict, outputs: Optional[tuple] = None) -> tuple:
        if outputs is not None:
            return outputs
        loss, _, _ = self.forward(batch)
        return loss, None, None

    def get_metrics(self, is_train: bool = False) -> dict:
        return {"loss": DistLoss()}

    def update_metric(self, batch: dict, outputs: tuple, metric) -> None:
        metric.update(outputs[0])

    # ------------------------------------------------------------------ sampler (model.py:231-353)
    def edm_sampler_loop(self, x: torch.Tensor, y: torch.Tensor, steps: Optional[int] = None, cfg: float = 1.0, **kwargs):
        """Heun sampler with fp64 state (model.py:232-297); every denoiser call goes through the fused kernels.  Where
        _sampler_graph_eligible holds, the whole loop runs as replays of captured CUDA graphs (engine.SamplerGraph),
        bit-identical to the eager loop and drawing the same random numbers; everywhere else the eager loop runs."""
        fwd = partial(self.dit.forward, cfg=cfg) if cfg > 1.0 else self.dit.forward
        graph = self._sampler_graph_eligible(fwd, x, y, kwargs)  # in the caller's grad mode
        with torch.no_grad():
            e = self.edm_config
            n = e.num_steps if steps is None else steps
            i = torch.arange(n, dtype=torch.float64, device=x.device)
            t_steps = (e.sigma_max ** (1 / e.rho) + i / (n - 1) * (e.sigma_min ** (1 / e.rho) - e.sigma_max ** (1 / e.rho))) ** e.rho
            t_steps = torch.cat([torch.as_tensor(t_steps), torch.zeros_like(t_steps[:1])])
            x_next = x.to(torch.float64) * t_steps[0]
            if graph:
                return self._heun_graph(x_next, t_steps, y, cfg if cfg > 1.0 else 1.0, n)
            # the caption is the same tensor for all 2n-1 denoiser calls: its stem and the 34 cross-attention K/V projections
            # are computed once (engine.prompt_cache) -- the reference recomputes them per call (dit.py:481-485,
            # utils.py:116-129)
            self._prompt_memo = {"y": y, "cfg": cfg if cfg > 1.0 else 1.0, "pc": None, "cap": None} if self.cache_prompt else None
            try:
                return self._heun(x_next, t_steps, y, fwd, n, **kwargs)
            finally:
                self._prompt_memo = None

    def _sampler_graph_eligible(self, fwd, x, y, kwargs) -> bool:
        """The rule for the CUDA-graph sampler: the CUDA ops, the model's own DiT as the denoiser with no extra keyword
        arguments, the prompt cache on, model_forward_wrapper not overridden, no gradient wanted for x or y, and
        sampler_graph not switched off.  Anything else keeps the eager loop, whose semantics it then defines."""
        from ..ops import CudaOps
        if not (self.sampler_graph and self.cache_prompt) or kwargs or not self._own_forward(fwd)[0]:
            return False
        if type(self).model_forward_wrapper is not LatentDiffusion.model_forward_wrapper:
            return False
        if torch.is_grad_enabled() and any(torch.is_tensor(v) and v.requires_grad for v in (x, y)):
            return False
        return isinstance(self.dit.engine.ops, CudaOps)

    def _heun_schedule(self, t_steps, n):
        """(t_steps, t_hat) on the host in fp64: the values _heun computes per step, the S_churn window's gamma decided
        with the same expressions, once per run."""
        e = self.edm_config
        t_cpu = t_steps.cpu()
        t_hat = []
        for t_cur in t_cpu[:n]:
            gamma = min(e.S_churn / n, np.sqrt(2) - 1) if e.S_min <= t_cur <= e.S_max else 0
            t_hat.append(torch.as_tensor(t_cur + gamma * t_cur))
        return t_cpu, torch.stack(t_hat) if t_hat else torch.zeros(0, dtype=torch.float64)

    def _predraw_noise(self, x_cur, n):
        """The n draws self.randn_like(x_cur) of the eager loop, in its order (the denoiser draws nothing at mask ratio
        0), so that the values and the generator state afterwards are the eager loop's."""
        return [self.randn_like(x_cur) for _ in range(n)]

    def _heun_graph(self, x_next, t_steps, y, cfg, n):
        t_cpu, t_hat = self._heun_schedule(t_steps, n)
        noise = self._predraw_noise(x_next, n)
        cap = self.dit._caption_f16(y)
        B = x_next.shape[0]
        eng = self.dit.engine
        sg = eng.sampler(B, cfg != 1.0, tuple(x_next.shape[1:]), tuple(cap.shape[1:]))
        return sg.run(x_next, t_cpu, t_hat, noise, cap, cfg, self.edm_config.S_noise, self._edm_scalars(),
                      debug=self.sampler_debug)

    def _heun(self, x_next, t_steps, y, fwd, n, **kwargs):
        e = self.edm_config
        for k, (t_cur, t_next) in enumerate(zip(t_steps[:-1], t_steps[1:])):
            x_cur = x_next
            gamma = min(e.S_churn / n, np.sqrt(2) - 1) if e.S_min <= t_cur <= e.S_max else 0
            t_hat = torch.as_tensor(t_cur + gamma * t_cur)
            x_hat = x_cur + (t_hat ** 2 - t_cur ** 2).sqrt() * e.S_noise * self.randn_like(x_cur)
            den = self.model_forward_wrapper(x_hat.to(torch.float32), t_hat.to(torch.float32), y, fwd, mask_ratio=0,
                                             **kwargs)["sample"]
            if self.sampler_debug is not None:
                self.sampler_debug(k, 0, den)
            den = den.to(torch.float64)
            d_cur = (x_hat - den) / t_hat
            x_next = x_hat + (t_next - t_hat) * d_cur
            if k < n - 1:
                den = self.model_forward_wrapper(x_next.to(torch.float32), t_next.to(torch.float32), y, fwd,
                                                 mask_ratio=0, **kwargs)["sample"]
                if self.sampler_debug is not None:
                    self.sampler_debug(k, 1, den)
                den = den.to(torch.float64)
                d_prime = (x_next - den) / t_next
                x_next = x_hat + (t_next - t_hat) * (0.5 * d_cur + 0.5 * d_prime)
        return x_next.to(torch.float32)

    @torch.no_grad()
    def generate(self, prompt: Optional[list] = None, tokenized_prompts: Optional[torch.LongTensor] = None,
                 attention_mask: Optional[torch.LongTensor] = None, guidance_scale: Optional[float] = 5.0,
                 num_inference_steps: Optional[int] = 30, seed: Optional[int] = None,
                 return_only_latents: Optional[bool] = False, **kwargs) -> torch.Tensor:
        assert prompt or tokenized_prompts is not None, "Must provide either prompt or tokenized prompts"
        device = self.vae.device
        gen = torch.Generator(device=device)
        if seed:
            gen = gen.manual_seed(seed)
        if tokenized_prompts is None:
            out = self.tokenizer.tokenize(prompt)
            tokenized_prompts = out["input_ids"]
            attention_mask = out["attention_mask"] if "attention_mask" in out else None
        text_embeddings = self.text_encoder.encode(
            tokenized_prompts.to(device), attention_mask=attention_mask.to(device) if attention_mask is not None else None)[0]
        latents = torch.randn((len(text_embeddings), self.dit.in_channels, self.latent_res, self.latent_res),
                              device=device, generator=gen)
        latents = self.edm_sampler_loop(latents, text_embeddings, num_inference_steps, cfg=guidance_scale)
        if return_only_latents:
            return latents
        latents = 1 / self.latent_scale * latents
        image = self.vae.decode(latents.to(DATA_TYPES[self.dtype])).sample
        return (image / 2 + 0.5).clamp(0, 1).float().detach()


def create_latent_diffusion(vae_name: str = "stabilityai/stable-diffusion-xl-base-1.0",
                            text_encoder_name: str = "openclip:hf-hub:apple/DFN5B-CLIP-ViT-H-14-378",
                            dit_arch: str = "MicroDiT_XL_2", latent_res: int = 32, in_channels: int = 4,
                            pos_interp_scale: float = 1.0, dtype: str = "bfloat16", precomputed_latents: bool = True,
                            p_mean: float = -0.6, p_std: float = 1.2, train_mask_ratio: float = 0.0,
                            vae=None, text_encoder=None, tokenizer=None) -> LatentDiffusion:
    """Factory with the reference's signature (model.py:356-405).  The frozen VAE / text encoder / tokenizer
    are outside the hot path: they are loaded exactly as the reference does when `diffusers` / `open_clip` are
    available, or may be passed in (e.g. stubs when training from precomputed latents, which train.py:25 asserts)."""
    s, d = text_encoder_embedding_format(text_encoder_name)
    dit = getattr(model_zoo, dit_arch)(input_size=latent_res, caption_channels=d, pos_interp_scale=pos_interp_scale,
                                       in_channels=in_channels)
    if vae is None:
        from diffusers import AutoencoderKL  # noqa: WPS433 (frozen encoder, not on the hot path)
        vae = AutoencoderKL.from_pretrained(vae_name, subfolder=None if vae_name == "ostris/vae-kl-f8-d16" else "vae",
                                            torch_dtype=DATA_TYPES[dtype], pretrained=True)
    if text_encoder is None or tokenizer is None:
        from .frozen import UniversalTextEncoder, UniversalTokenizer
        text_encoder = text_encoder or UniversalTextEncoder(text_encoder_name, dtype=dtype, pretrained=True)
        tokenizer = tokenizer or UniversalTokenizer(text_encoder_name)
    return LatentDiffusion(dit=dit, vae=vae, text_encoder=text_encoder, tokenizer=tokenizer,
                           precomputed_latents=precomputed_latents, dtype=dtype, latent_res=latent_res, p_mean=p_mean,
                           p_std=p_std, train_mask_ratio=train_mask_ratio)


class PrecomputedLatentStubs:
    """Stand-ins for the frozen VAE / text encoder when every batch carries precomputed latents (train.py:25):
    only `.config.scaling_factor`, `.requires_grad_`, `.to`, `.device` are ever touched."""

    class _VAE:
        class config:  # noqa: N801
            scaling_factor = 0.13025
        device = torch.device("cpu")

        def requires_grad_(self, flag):
            return self

        def to(self, device):
            self.device = torch.device(device)
            return self

    class _Text:
        def requires_grad_(self, flag):
            return self

        def to(self, device):
            return self

    class _Tok:
        model_max_length = 77

        def tokenize(self, captions):
            raise RuntimeError("no tokenizer: this model was built for precomputed latents only")

    @classmethod
    def make(cls):
        return cls._VAE(), cls._Text(), cls._Tok()
