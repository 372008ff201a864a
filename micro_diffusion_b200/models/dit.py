"""`model.dit`: the MicroDiT denoiser behind the reference's module surface.

Same constructor arguments, attribute names, factories and state_dict (476 parameters + `pos_embed`,
`mask_token`; SURVEY.md section 8b) as reference micro_diffusion/models/dit.py, but the module holds no
compute: parameters are views into one flat fp32 buffer (`params.ParamStore`) and `forward` hands raw
device pointers to the sm_90a kernels through `engine.Engine`.  Gradients come from the hand-written CUDA
backward: `LatentDiffusion.forward` drives it for the fused EDM loss (models/model.py), and `DiT.forward` under grad
mode records one autograd node (`_DiTForwardFn`) whose backward runs the same backward from an arbitrary output
cotangent and returns the gradients of x, t and y.  Under no_grad `DiT.forward` is the plain inference entry.
"""
from __future__ import annotations

from typing import List, Optional

import torch
import torch.nn as nn
from torch.autograd.function import once_differentiable

from ..arch import DiTConfig, micro_dit_tiny_2_kwargs, micro_dit_xl_2_kwargs
from ..engine import Engine
from ..params import ParamLayout, ParamStore
from .utils import get_2d_sincos_pos_embed


class _Node(nn.Module):
    """Name-space container so that parameter paths (blocks.3.attn.qkv.weight ...) match the reference."""

    def __getitem__(self, i):
        return getattr(self, str(i))

    def __len__(self):
        return len(self._modules)

    def __iter__(self):
        return iter(self._modules.values())


def _trunc_normal_(t: torch.Tensor, std: float, gen=None):
    # nn.init.trunc_normal_(mean=0, std, a=-2, b=2): with std ~0.02 the +-2 cut never binds in practice,
    # but keep the semantics.
    with torch.no_grad():
        t.normal_(0.0, std, generator=gen).clamp_(-2.0, 2.0)


class _DiTForwardFn(torch.autograd.Function):
    """F = DiT.forward_without_cfg(x, t, y)["sample"] with the forward and its vector-Jacobian product run by the engine.

    `anchor` is the DiT's gradient anchor when parameter gradients are wanted (they accumulate into the flat buffer behind
    `p.grad`, like the fused loss) and None when every parameter is frozen.  x f32 and t f32 [B] arrive already cast and
    broadcast by the caller, so autograd handles those; the fp16 storage cast of y happens in here and its gradient is
    returned in y's own dtype (a straight-through cast, without rounding the gradient to fp16)."""

    @staticmethod
    def forward(ctx, anchor, dit, x, t, y, mask_ratio, mask_noise):
        fx, mask, c = dit.engine.forward_raw(x, t, dit._caption_f16(y), mask_ratio, mask_noise, keep=True)
        ctx.dit, ctx.c, ctx.param_grads = dit, c, anchor is not None
        ctx.y_shape, ctx.y_dtype = y.shape, y.dtype
        if mask is not None:
            ctx.mark_non_differentiable(mask)
        return fx, mask

    @staticmethod
    @once_differentiable
    def backward(ctx, dfx, dmask=None):
        dit, c = ctx.dit, ctx.c
        if c is None:
            raise RuntimeError("DiT backward: no saved activations (backward called twice through the same forward)")
        want_dx, want_dt, want_dy = ctx.needs_input_grad[2:5]
        if ctx.param_grads:
            dit.prepare_grads()
        dF = dfx.detach().to(torch.float32).contiguous()
        dx, dt, dy = dit.engine.backward_output(c, dF, param_grads=ctx.param_grads, want_dx=want_dx, want_dt=want_dt,
                                                want_dy=want_dy)
        ctx.c = None  # free the saved activations
        if dy is not None:
            dy = dy.reshape(ctx.y_shape).to(ctx.y_dtype)
        return None, None, dx, dt, dy, None, None


class DiT(nn.Module):
    def __init__(self, input_size: int = 32, patch_size: int = 2, in_channels: int = 4, dim: int = 1152,
                 depth: int = 28, head_dim: int = 64, multiple_of: int = 256, caption_channels: int = 1024,
                 pos_interp_scale: float = 1.0, norm_eps: float = 1e-6, depth_init: bool = True,
                 qkv_multipliers: List[float] = (1.0,), ffn_multipliers: List[float] = (4.0,),
                 use_patch_mixer: bool = True, patch_mixer_depth: int = 4, patch_mixer_dim: int = 512,
                 patch_mixer_qkv_ratio: float = 1.0, patch_mixer_mlp_ratio: float = 1.0, use_bias: bool = True,
                 num_experts: int = 8, expert_capacity: int = 1, experts_every_n: int = 2, ops_factory=None):
        super().__init__()
        self.cfg = DiTConfig(input_size=input_size, patch_size=patch_size, in_channels=in_channels, dim=dim, depth=depth,
                             head_dim=head_dim, multiple_of=multiple_of, caption_channels=caption_channels,
                             pos_interp_scale=pos_interp_scale, norm_eps=norm_eps, depth_init=depth_init,
                             qkv_multipliers=tuple(qkv_multipliers), ffn_multipliers=tuple(ffn_multipliers),
                             use_patch_mixer=use_patch_mixer, patch_mixer_depth=patch_mixer_depth,
                             patch_mixer_dim=patch_mixer_dim, patch_mixer_qkv_ratio=patch_mixer_qkv_ratio,
                             patch_mixer_mlp_ratio=patch_mixer_mlp_ratio, use_bias=use_bias, num_experts=num_experts,
                             expert_capacity=expert_capacity, experts_every_n=experts_every_n)
        if not use_patch_mixer:
            raise NotImplementedError("use_patch_mixer=False is not supported: the reference cannot build it either (its "
                                      "initialize_weights reads self.patch_mixer, which only exists with the mixer, "
                                      "dit.py:612)")
        # attributes the reference exposes (dit.py:303-309) and LatentDiffusion / callbacks read
        self.input_size, self.in_channels, self.out_channels = input_size, in_channels, in_channels
        self.patch_size, self.head_dim, self.pos_interp_scale = patch_size, head_dim, pos_interp_scale
        self.use_patch_mixer = use_patch_mixer
        self.base_size = input_size // patch_size
        self._ops_factory = ops_factory  # test hook: inject oracle.emu_ops.EmuOps; default = CUDA kernels
        self._layout = ParamLayout(self.cfg)
        self._store: Optional[ParamStore] = None
        self._engine: Optional[Engine] = None
        self._anchor = None
        self._flat_guard = False

        # buffers first: the reference's state_dict starts with pos_embed, mask_token (dit.py:319,440-443)
        self.register_buffer("pos_embed", torch.zeros(1, self.cfg.num_patches, dim))
        self.register_buffer("mask_token", torch.zeros(1, 1, patch_size ** 2 * self.out_channels))
        self._param_names: List[str] = []
        flat = torch.zeros(self._layout.total, dtype=torch.float32)
        self._flat_cpu_init = flat
        for name, shape in self.cfg.param_specs():
            off, shp = self._layout.slots[name]
            n = 1
            for d in shp:
                n *= d
            self._register(name, nn.Parameter(flat[off:off + n].view(shp)))
        self.x_embedder.patch_size = (patch_size, patch_size)
        self.x_embedder.num_patches = self.cfg.num_patches
        self.initialize_weights()

    # ------------------------------------------------------------------ registration / storage
    def _register(self, name: str, param: nn.Parameter):
        parts = name.split(".")
        node = self
        for p in parts[:-1]:
            if p not in node._modules:
                node.add_module(p, _Node())
            node = node._modules[p]
        node.register_parameter(parts[-1], param)
        self._param_names.append(name)

    def _named(self):
        return {n: p for n, p in self.named_parameters()}

    def _bind(self, device=None, force=False):
        """(Re)point every parameter at the flat device buffer; called lazily and after .to()/.cuda()."""
        params = self._named()
        first = params[self._param_names[0]]
        device = torch.device(device) if device is not None else first.device
        st = self._store
        if not force and st is not None and st.device == device:
            off, shp = self._layout.slots[self._param_names[0]]
            if first.data_ptr() == st.p[self._param_names[0]].data_ptr():
                return st
        ops = self._make_ops(device)
        new = ParamStore(self._layout, device, getattr(ops, "lowp_dtype", torch.bfloat16))
        with torch.no_grad():
            for n in self._param_names:
                new.p[n].copy_(params[n].data.to(device=device, dtype=torch.float32))
                had_grad = params[n].grad is not None
                if had_grad:
                    new.g[n].copy_(params[n].grad.to(device=device, dtype=torch.float32))
                params[n].data = new.p[n]
                params[n].grad = new.g[n] if had_grad else None
        self._store = new
        self._flat_cpu_init = None
        self._engine = Engine(self.cfg, new, ops)
        self._plist = [params[n] for n in self._param_names]
        self._dirty = self.__dict__.get("_dirty", 0) + 1
        self._engine.weights_token = self._weights_token
        self._anchor = torch.zeros(1, device=device, requires_grad=True)
        return new

    def _make_ops(self, device):
        if self._ops_factory is not None:
            return self._ops_factory(device)
        from ..ops import CudaOps  # raises loudly on CPU or when the library is missing
        return CudaOps(device)

    def _apply(self, fn, *args, **kwargs):
        out = super()._apply(fn, *args, **kwargs)
        if self._store is not None:  # storage moved underneath us: re-flatten on the new device
            self._bind(force=True)
        return out

    def _weights_token(self):
        # every in-place write through a Parameter (optimizer step, load_state_dict, clip_grad...) bumps its
        # autograd version counter; writes through `.data` do not -- call mark_weights_dirty() after those.
        return (self._dirty, sum(p._version for p in self._plist))

    def mark_weights_dirty(self):
        self._dirty = self.__dict__.get("_dirty", 0) + 1  # legal before the first bind

    @property
    def engine(self) -> Engine:
        self._bind()
        eng = self._engine
        eng.pos_embed = self.pos_embed.detach().float().contiguous()
        eng.mask_token = self.mask_token.detach().float().contiguous()
        return eng

    @property
    def store(self) -> ParamStore:
        return self._bind()

    def prepare_grads(self):
        """Make every `p.grad` a view of the flat gradient buffer (zeroing segments whose grad was None)."""
        st = self._bind()
        params = self._named()
        missing = [n for n in self._param_names if params[n].grad is None]
        if len(missing) == len(self._param_names):
            st.grad.zero_()
        for n in self._param_names:
            p = params[n]
            if p.grad is None:
                if len(missing) != len(self._param_names):
                    st.g[n].zero_()
                p.grad = st.g[n]
            elif p.grad.data_ptr() != st.g[n].data_ptr():
                st.g[n].copy_(p.grad)
                p.grad = st.g[n]

    # ------------------------------------------------------------------ init (dit.py:577-627)
    def initialize_weights(self) -> None:
        cfg = self.cfg
        P = self._named()
        with torch.no_grad():
            for n, p in P.items():
                if p.dim() == 2 and not n.endswith("mlp.gate.weight"):  # _basic_init: xavier on every nn.Linear
                    nn.init.xavier_uniform_(p)
                elif p.dim() == 2:
                    nn.init.xavier_uniform_(p)
                elif n.endswith(".bias"):
                    p.zero_()
                elif p.dim() == 1:
                    p.fill_(1.0)  # LayerNorm gains
            pe = get_2d_sincos_pos_embed(cfg.dim, cfg.grid, pos_interp_scale=cfg.pos_interp_scale, base_size=self.base_size)
            self.pos_embed.copy_(torch.from_numpy(pe).float().unsqueeze(0))
            w = P["x_embedder.proj.weight"]
            nn.init.xavier_uniform_(w.view(w.shape[0], -1))
            # nn.Conv2d's default bias init survives in the reference (_basic_init only touches nn.Linear)
            bound = 1.0 / (w.shape[1] * w.shape[2] * w.shape[3]) ** 0.5
            P["x_embedder.proj.bias"].uniform_(-bound, bound)
            for n in ("t_embedder.mlp.0.weight", "t_embedder.mlp.2.weight", "pooled_y_emb_process.fc1.weight",
                      "pooled_y_emb_process.fc2.weight", "y_embedder.y_proj.fc1.weight", "y_embedder.y_proj.fc2.weight"):
                P[n].normal_(0.0, 0.02)
            for b in cfg.all_blocks():  # DiTBlock.custom_init (dit.py:241-246)
                pre = b.name
                _trunc_normal_(P[pre + ".attn.qkv.weight"], 0.02)
                _trunc_normal_(P[pre + ".attn.proj.weight"], b.init_std)
                _trunc_normal_(P[pre + ".cross_attn.q_linear.weight"], 0.02)
                _trunc_normal_(P[pre + ".cross_attn.kv_linear.weight"], 0.02)
                _trunc_normal_(P[pre + ".cross_attn.proj.weight"], b.init_std)
                if b.moe:
                    _trunc_normal_(P[pre + ".mlp.gate.weight"], 0.02)
                    _trunc_normal_(P[pre + ".mlp.w1"], 0.02)
                    _trunc_normal_(P[pre + ".mlp.w2"], b.init_std)
                else:
                    _trunc_normal_(P[pre + ".mlp.w1.weight"], 0.02)
                    _trunc_normal_(P[pre + ".mlp.w2.weight"], b.init_std)
                    _trunc_normal_(P[pre + ".mlp.w3.weight"], b.init_std)
                P[pre + ".adaLN_modulation.1.weight"].zero_()
            # AttentionBlockPromptEmbedding.custom_init() with the default init_std=0.02, then zeroed outputs
            _trunc_normal_(P["y_emb_preprocess.attn.qkv.weight"], 0.02)
            _trunc_normal_(P["y_emb_preprocess.mlp.w1.weight"], 0.02)
            _trunc_normal_(P["y_emb_preprocess.mlp.w2.weight"], 0.02)
            P["y_emb_preprocess.attn.proj.weight"].zero_()
            P["y_emb_preprocess.mlp.w3.weight"].zero_()
            P["final_layer.adaLN_modulation.1.weight"].zero_()
            P["final_layer.linear.weight"].zero_()

    # ------------------------------------------------------------------ forward (dit.py:455-564)
    def forward_without_cfg(self, x, t, y, mask_ratio: float = 0, **kwargs) -> dict:
        """Differentiable like the reference's: under grad mode, when x, t, y or the parameters require grad, the output
        carries one autograd node whose backward is the engine's hand-derived backward.  Otherwise (e.g. under no_grad)
        nothing is saved."""
        if torch.is_grad_enabled():
            param_grads = self._param_grad_mode()
            if param_grads or any(torch.is_tensor(v) and v.requires_grad for v in (x, t, y)):
                self.engine  # bind storage / anchor before the autograd node is built
                B = x.shape[0]
                x = x.float().contiguous()
                t = t.float().reshape(-1).expand(B).contiguous()
                noise = None
                if mask_ratio > 0:
                    noise = torch.rand(B, self.cfg.num_patches, device=x.device)  # get_mask (utils.py:390)
                fx, mask = _DiTForwardFn.apply(self._anchor if param_grads else None, self, x, t, y, float(mask_ratio),
                                               noise)
                return {"sample": fx, "mask": mask}
        return self._forward_inference(x, t, y, mask_ratio)

    @torch.no_grad()
    def _forward_inference(self, x, t, y, mask_ratio):
        eng = self.engine
        B = x.shape[0]
        x = x.float().contiguous()
        t = t.float().reshape(-1).expand(B).contiguous()
        cap = self._caption_f16(y)
        noise = None
        if mask_ratio > 0:
            noise = torch.rand(B, self.cfg.num_patches, device=x.device)  # get_mask (utils.py:390)
        fx, mask = eng.forward_raw(x, t, cap, mask_ratio, noise)
        return {"sample": fx, "mask": mask}

    def _param_grad_mode(self) -> bool:
        """True when every parameter requires grad, False when none does; per-parameter freezing is not supported."""
        req = {p.requires_grad for p in self.parameters()}
        if len(req) > 1:
            raise NotImplementedError("DiT: some parameters require grad and some do not. The CUDA backward computes the "
                                      "gradients of all parameters or of none: set requires_grad on all of them, or on "
                                      "none (input gradients only).")
        return req.pop()

    def forward_with_cfg(self, x, t, y, cfg: float = 1.0, mask_ratio: float = 0, **kwargs) -> dict:
        x = torch.cat([x, x], 0)
        y = torch.cat([y, torch.zeros_like(y)], 0)
        if len(t) != 1:
            t = torch.cat([t, t], 0)
        eps = self.forward_without_cfg(x, t, y, mask_ratio, **kwargs)["sample"]
        cond_eps, uncond_eps = torch.split(eps, len(eps) // 2, dim=0)
        return {"sample": uncond_eps + cfg * (cond_eps - uncond_eps)}

    def forward(self, x, t, y, cfg: float = 1.0, **kwargs) -> dict:
        if cfg != 1.0:
            return self.forward_with_cfg(x, t, y, cfg, **kwargs)
        return self.forward_without_cfg(x, t, y, **kwargs)

    @staticmethod
    def _caption_f16(y):
        if y.dtype != torch.float16:
            y = y.to(torch.float16)  # storage-format cast of an input (the loader delivers fp16, latents_loader.py:52-55)
        return y.contiguous()

    def unpatchify(self, x):
        """(N, T, p*p*C) -> (N, C, H, W)  (dit.py:566-575); host-side utility, not on the hot path."""
        c, p = self.out_channels, self.patch_size
        h = w = int(x.shape[1] ** 0.5)
        assert h * w == x.shape[1]
        x = x.reshape(x.shape[0], h, w, p, p, c)
        return x.permute(0, 5, 1, 3, 2, 4).reshape(x.shape[0], c, h * p, w * p)


def MicroDiT_Tiny_2(caption_channels: int = 1024, qkv_ratio=(0.5, 1.0), mlp_ratio=(0.5, 4.0), pos_interp_scale: float = 1.0,
                    input_size: int = 32, num_experts: int = 8, expert_capacity: float = 2.0, experts_every_n: int = 2,
                    in_channels: int = 4, **kwargs) -> DiT:
    return DiT(**micro_dit_tiny_2_kwargs(caption_channels, qkv_ratio, mlp_ratio, pos_interp_scale, input_size,
                                         num_experts, expert_capacity, experts_every_n, in_channels), **kwargs)


def MicroDiT_XL_2(caption_channels: int = 1024, qkv_ratio=(0.5, 1.0), mlp_ratio=(0.5, 4.0), pos_interp_scale: float = 1.0,
                  input_size: int = 32, num_experts: int = 8, expert_capacity: float = 2.0, experts_every_n: int = 2,
                  in_channels: int = 4, **kwargs) -> DiT:
    return DiT(**micro_dit_xl_2_kwargs(caption_channels, qkv_ratio, mlp_ratio, pos_interp_scale, input_size,
                                       num_experts, expert_capacity, experts_every_n, in_channels), **kwargs)
