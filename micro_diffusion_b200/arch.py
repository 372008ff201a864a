"""Architecture arithmetic of the MicroDiT denoiser: constructor arguments -> per-block widths and the
ordered parameter list (names and shapes identical to the reference state_dict).

Mirrors the sizing rules of the reference constructors, citing them:
  DiT.__init__                 micro_diffusion/models/dit.py:277-453
  DiTBlock.__init__            dit.py:171-230   (qkv hidden width, mlp hidden width)
  FeedForward.__init__         dit.py:72-86     (2/3 rule, round up to multiple_of)
  FeedForwardECMoe.__init__    dit.py:107-124
  MicroDiT_Tiny_2 / _XL_2      dit.py:630-709   (np.linspace ratios)
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Sequence, Tuple

import numpy as np


def _round_up(x: int, m: int) -> int:
    return m * ((x + m - 1) // m)


@dataclass(frozen=True)
class BlockSpec:
    name: str          # "patch_mixer.3" / "blocks.17"
    dim: int           # block width D
    attn_dim: int      # self-attention hidden width h (multiple of 2*head_dim)
    heads: int         # h / head_dim
    xheads: int        # cross-attention heads (= D / head_dim, compress_xattn=False)
    moe: bool
    ffn_dim: int       # f
    init_std: float    # weight_init_std of the block (dit.py:227-230)


@dataclass
class DiTConfig:
    input_size: int = 32
    patch_size: int = 2
    in_channels: int = 4
    dim: int = 1152
    depth: int = 28
    head_dim: int = 64
    multiple_of: int = 256
    caption_channels: int = 1024
    pos_interp_scale: float = 1.0
    norm_eps: float = 1e-6
    depth_init: bool = True
    qkv_multipliers: Sequence[float] = (1.0,)
    ffn_multipliers: Sequence[float] = (4.0,)
    use_patch_mixer: bool = True
    patch_mixer_depth: int = 4
    patch_mixer_dim: int = 512
    patch_mixer_qkv_ratio: float = 1.0
    patch_mixer_mlp_ratio: float = 1.0
    use_bias: bool = True
    num_experts: int = 8
    expert_capacity: float = 1
    experts_every_n: int = 2
    freq_dim: int = 512  # TimestepEmbedder.frequency_embedding_size (utils.py:256)

    # derived
    mixer_blocks: List[BlockSpec] = field(default_factory=list, init=False)
    blocks: List[BlockSpec] = field(default_factory=list, init=False)

    def __post_init__(self):
        assert self.dim % self.head_dim == 0, "Hidden dimension must be divisible by head dim"
        qm, fm = list(self.qkv_multipliers), list(self.ffn_multipliers)
        assert len(qm) == len(fm)
        if len(fm) == self.depth:
            qkv_ratios, mlp_ratios = qm, fm
        else:  # spread the multipliers over equal partitions (dit.py:397-407)
            n = len(fm)
            assert self.depth % n == 0, "number of blocks should be divisible by number of splits"
            per = self.depth // n
            qkv_ratios = [m for m in qm for _ in range(per)]
            mlp_ratios = [m for m in fm for _ in range(per)]
        self.mixer_blocks = []
        if self.use_patch_mixer:
            for i in range(self.patch_mixer_depth):
                moe = i >= 1 and (i + 1) % self.experts_every_n == 0  # dit.py:346-353
                self.mixer_blocks.append(self._block(f"patch_mixer.{i}", self.patch_mixer_dim, self.patch_mixer_qkv_ratio,
                                                     self.patch_mixer_mlp_ratio, moe, depth_init=False, layer_id=0))
        self.blocks = []
        for i in range(self.depth):
            moe = i < self.depth - 1 and (i + 1) % self.experts_every_n == 0  # no MoE in the last block (dit.py:409-417)
            self.blocks.append(self._block(f"blocks.{i}", self.dim, float(qkv_ratios[i]), float(mlp_ratios[i]), moe,
                                           depth_init=self.depth_init, layer_id=i))

    def _block(self, name, dim, qkv_ratio, mlp_ratio, moe, depth_init, layer_id) -> BlockSpec:
        hd2 = self.head_dim * 2
        attn_dim = hd2 * ((int(dim * qkv_ratio) + hd2 - 1) // hd2) if qkv_ratio != 1 else dim
        mlp_hidden = int(dim * mlp_ratio)
        if moe:
            ffn = _round_up(mlp_hidden, self.multiple_of)
        else:
            ffn = _round_up(int(2 * mlp_hidden / 3), self.multiple_of)
        std = 0.02 / (2 * (layer_id + 1)) ** 0.5 if depth_init else 0.02 / (2 * self.depth) ** 0.5
        assert attn_dim % self.head_dim == 0 and dim % self.head_dim == 0
        return BlockSpec(name, dim, attn_dim, attn_dim // self.head_dim, dim // self.head_dim, moe, ffn, std)

    # ------------------------------------------------------------------ sizes
    @property
    def grid(self) -> int:
        return self.input_size // self.patch_size

    @property
    def num_patches(self) -> int:
        return self.grid * self.grid

    @property
    def patch_dim(self) -> int:
        return self.patch_size * self.patch_size * self.in_channels

    @property
    def mixer_dim(self) -> int:
        return self.patch_mixer_dim if self.use_patch_mixer else self.dim

    @property
    def has_mixer_maps(self) -> bool:
        return self.use_patch_mixer and self.patch_mixer_dim != self.dim

    @property
    def prompt_ffn_dim(self) -> int:  # y_emb_preprocess: FeedForward(dim, int(dim*4.0)) (dit.py:328-335)
        return _round_up(int(2 * int(self.dim * 4.0) / 3), self.multiple_of)

    def all_blocks(self) -> List[BlockSpec]:
        return [*self.mixer_blocks, *self.blocks]

    # ------------------------------------------------------------------ parameter list
    def _linear(self, name: str, out_f: int, in_f: int) -> List[Tuple[str, Tuple[int, ...]]]:
        """nn.Linear(in_f, out_f, bias=use_bias): the weight, then its bias when the model has biases."""
        return [(name + ".weight", (out_f, in_f))] + ([(name + ".bias", (out_f,))] if self.use_bias else [])

    def block_param_specs(self, b: BlockSpec) -> List[Tuple[str, Tuple[int, ...]]]:
        D, h, f, E = b.dim, b.attn_dim, b.ffn_dim, self.num_experts
        p, lin = b.name, self._linear
        out = [(f"{p}.norm1.weight", (D,)), *lin(f"{p}.attn.qkv", 3 * h, D), *lin(f"{p}.attn.proj", D, h),
               *lin(f"{p}.cross_attn.q_linear", D, D), *lin(f"{p}.cross_attn.kv_linear", 2 * D, D),
               *lin(f"{p}.cross_attn.proj", D, D), (f"{p}.norm2.weight", (D,)), (f"{p}.norm3.weight", (D,))]
        if b.moe:  # the expert banks are raw parameters and the gate is bias-free whatever use_bias says (dit.py:107-124)
            out += [(f"{p}.mlp.w1", (E, D, f)), (f"{p}.mlp.w2", (E, f, D)), (f"{p}.mlp.gate.weight", (E, D))]
        else:
            out += [*lin(f"{p}.mlp.w1", f, D), *lin(f"{p}.mlp.w2", f, D), *lin(f"{p}.mlp.w3", D, f)]
        out += [(f"{p}.adaLN_modulation.1.weight", (6 * D, self.dim)), (f"{p}.adaLN_modulation.1.bias", (6 * D,))]
        return out

    def param_specs(self) -> List[Tuple[str, Tuple[int, ...]]]:
        """(name, shape) of every trainable parameter, in the reference's state_dict order.  use_bias=True adds the bias
        of every block linear, of the prompt block's attention / SwiGLU and of the mixer maps (dit.py:39-51,84-86,202-219,
        377-388), each right after its weight."""
        D, C, p, Dc = self.dim, self.in_channels, self.patch_size, self.caption_channels
        lin = self._linear
        fp = self.prompt_ffn_dim
        s: List[Tuple[str, Tuple[int, ...]]] = [
            ("x_embedder.proj.weight", (D, C, p, p)), ("x_embedder.proj.bias", (D,)),
            ("t_embedder.mlp.0.weight", (D, self.freq_dim)), ("t_embedder.mlp.0.bias", (D,)),
            ("t_embedder.mlp.2.weight", (D, D)), ("t_embedder.mlp.2.bias", (D,)),
            ("y_embedder.y_proj.fc1.weight", (D, Dc)), ("y_embedder.y_proj.fc1.bias", (D,)),
            ("y_embedder.y_proj.norm.weight", (D,)),
            ("y_embedder.y_proj.fc2.weight", (D, D)), ("y_embedder.y_proj.fc2.bias", (D,)),
            ("y_emb_preprocess.norm1.weight", (D,)), *lin("y_emb_preprocess.attn.qkv", 3 * D, D),
            *lin("y_emb_preprocess.attn.proj", D, D), ("y_emb_preprocess.norm2.weight", (D,)),
            *lin("y_emb_preprocess.mlp.w1", fp, D), *lin("y_emb_preprocess.mlp.w2", fp, D),
            *lin("y_emb_preprocess.mlp.w3", D, fp),
            ("pooled_y_emb_process.fc1.weight", (D, D)), ("pooled_y_emb_process.fc1.bias", (D,)),
            ("pooled_y_emb_process.norm.weight", (D,)),
            ("pooled_y_emb_process.fc2.weight", (D, D)), ("pooled_y_emb_process.fc2.bias", (D,)),
        ]
        for b in self.mixer_blocks:
            s += self.block_param_specs(b)
        if self.has_mixer_maps:
            Dm = self.patch_mixer_dim
            s += [("patch_mixer_map_xin.0.weight", (D,)), *lin("patch_mixer_map_xin.1", Dm, D),
                  ("patch_mixer_map_xout.0.weight", (Dm,)), *lin("patch_mixer_map_xout.1", D, Dm),
                  ("patch_mixer_map_y.0.weight", (D,)), *lin("patch_mixer_map_y.1", Dm, D)]
        for b in self.blocks:
            s += self.block_param_specs(b)
        s += [("final_layer.linear.weight", (self.patch_dim, D)), ("final_layer.linear.bias", (self.patch_dim,)),
              ("final_layer.adaLN_modulation.1.weight", (2 * D, D)), ("final_layer.adaLN_modulation.1.bias", (2 * D,)),
              ("final_layer.norm_final.weight", (D,))]
        return s

    def buffer_specs(self) -> List[Tuple[str, Tuple[int, ...]]]:
        return [("pos_embed", (1, self.num_patches, self.dim)), ("mask_token", (1, 1, self.patch_dim))]


def micro_dit_xl_2_kwargs(caption_channels=1024, qkv_ratio=(0.5, 1.0), mlp_ratio=(0.5, 4.0), pos_interp_scale=1.0,
                          input_size=32, num_experts=8, expert_capacity=2.0, experts_every_n=2, in_channels=4):
    """MicroDiT_XL_2 (dit.py:671-709)."""
    depth = 28
    return dict(input_size=input_size, patch_size=2, in_channels=in_channels, dim=1024, depth=depth, head_dim=64,
                multiple_of=256, caption_channels=caption_channels, pos_interp_scale=pos_interp_scale, norm_eps=1e-6,
                depth_init=True,
                qkv_multipliers=tuple(np.linspace(qkv_ratio[0], qkv_ratio[1], num=depth, dtype=float)),
                ffn_multipliers=tuple(np.linspace(mlp_ratio[0], mlp_ratio[1], num=depth, dtype=float)),
                use_patch_mixer=True, patch_mixer_depth=6, patch_mixer_dim=768, patch_mixer_qkv_ratio=1.0,
                patch_mixer_mlp_ratio=4.0, use_bias=False, num_experts=num_experts, expert_capacity=expert_capacity,
                experts_every_n=experts_every_n)


def micro_dit_tiny_2_kwargs(caption_channels=1024, qkv_ratio=(0.5, 1.0), mlp_ratio=(0.5, 4.0), pos_interp_scale=1.0,
                            input_size=32, num_experts=8, expert_capacity=2.0, experts_every_n=2, in_channels=4):
    """MicroDiT_Tiny_2 (dit.py:630-668)."""
    depth = 16
    return dict(input_size=input_size, patch_size=2, in_channels=in_channels, dim=512, depth=depth, head_dim=32,
                multiple_of=256, caption_channels=caption_channels, pos_interp_scale=pos_interp_scale, norm_eps=1e-6,
                depth_init=True,
                qkv_multipliers=tuple(np.linspace(qkv_ratio[0], qkv_ratio[1], num=depth, dtype=float)),
                ffn_multipliers=tuple(np.linspace(mlp_ratio[0], mlp_ratio[1], num=depth, dtype=float)),
                use_patch_mixer=True, patch_mixer_depth=4, patch_mixer_dim=512, patch_mixer_qkv_ratio=1.0,
                patch_mixer_mlp_ratio=4.0, use_bias=False, num_experts=num_experts, expert_capacity=expert_capacity,
                experts_every_n=experts_every_n)
