"""Flat parameter / gradient storage for the MicroDiT denoiser.

All trainable tensors live in ONE fp32 buffer (and their gradients in a second one); the named
`nn.Parameter`s the reference exposes (`model.dit.named_parameters()`, the 476-entry state_dict) are
views into it.  That gives
  * one NCCL all-reduce (or a few buckets) over `grad` for the data-parallel gradient mean (SURVEY C1),
  * one fused AdamW launch over `flat` (SURVEY K13),
  * contiguous "GEMM groups": every adaLN weight stacked as one [sum(6D)+2D, dim] matrix so the 35
    per-block modulation linears (dit.py:233-235, utils.py:237) are a single GEMM, and w1|w2 of each
    SwiGLU stacked as one [2f, D] matrix (dit.py:84-89),
  * per-step bf16 operand copies (`wb`, same layout) and transposed copies (`wbt`) produced by
    md_cast_transpose -- what torch.autocast re-does on every call in the reference.
"""
from __future__ import annotations

import os

from dataclasses import dataclass
from typing import Dict, List, Tuple

import torch

from .arch import DiTConfig


def _numel(shape) -> int:
    n = 1
    for s in shape:
        n *= int(s)
    return n


@dataclass
class MatGroup:
    """A [batch, rows, cols] matrix living at `offset` in the flat buffers (one weight or a stacked group)."""
    name: str
    offset: int
    batch: int
    rows: int
    cols: int
    need_t: bool = True  # transposed bf16 copy needed (dgrad, or expert forward)

    @property
    def numel(self) -> int:
        return self.batch * self.rows * self.cols


class ParamLayout:
    """Name -> (offset, shape) in the flat buffers, plus the GEMM groups."""

    ALIGN = 8  # elements: 16 B for bf16 TMA bases, 32 B for fp32 vector loads
    RANGE_ALIGN = 1024  # boundaries of the gradient-exchange ranges: every range splits evenly over up to 128 ranks

    def __init__(self, cfg: DiTConfig):
        self.cfg = cfg
        specs = cfg.param_specs()
        ada_w = [s for s in specs if s[0].endswith("adaLN_modulation.1.weight")]
        ada_b = [s for s in specs if s[0].endswith("adaLN_modulation.1.bias")]
        # cross-attention K/V projections of all blocks of a stage act on the SAME caption tokens (dit.py:237,
        # utils.py:118): stacking their weights turns 28 (+6) medium GEMMs per direction into one large one.
        kv_m = [s for s in specs if s[0].startswith("patch_mixer.") and s[0].endswith("cross_attn.kv_linear.weight")]
        kv_b = [s for s in specs if s[0].startswith("blocks.") and s[0].endswith("cross_attn.kv_linear.weight")]
        # use_bias=True: the kv_linear biases of a stage follow its weight stack as one [nblk * 2D] vector (the bias of the
        # stacked GEMM), in block order
        kvb_m = [s for s in specs if s[0].startswith("patch_mixer.") and s[0].endswith("cross_attn.kv_linear.bias")]
        kvb_b = [s for s in specs if s[0].startswith("blocks.") and s[0].endswith("cross_attn.kv_linear.bias")]
        special = {s[0] for s in ada_w + ada_b + kv_m + kv_b + kvb_m + kvb_b}
        shapes = dict(specs)
        rest = []
        for name, shape in specs:
            if name in special or name.endswith("mlp.w1.bias"):
                continue  # w1.bias is placed after w2.weight below, so that the two weights stay adjacent (the w12 stack)
            rest.append((name, shape))
            b1 = name[: -len("w2.weight")] + "w1.bias"
            if name.endswith("mlp.w2.weight") and b1 in shapes:
                rest.append((b1, shapes[b1]))  # a SwiGLU's biases as one [b1 | b2] vector after the w1 | w2 weights
        self.order: List[Tuple[str, Tuple[int, ...]]] = ada_w + ada_b + kv_m + kvb_m + kv_b + kvb_b + rest
        self.reference_order = [s[0] for s in specs]
        self.slots: Dict[str, Tuple[int, Tuple[int, ...]]] = {}
        # The flat buffer is exchanged in a few contiguous ranges (train_step.GradReducer): "back" = the stacked backbone
        # K/V projection + everything from the first blocks.* / final_layer.* tensor to the end (final once the backbone
        # backward is done, needed last by the forward), "front" = the rest.  Range boundaries are padded to RANGE_ALIGN
        # so that each range reduce-scatters / all-gathers in equal 16-byte-aligned shares.
        def is_back_rest(nm):
            return nm.startswith("blocks.") or nm.startswith("final_layer.")
        bounds = set()
        if kv_b:
            bounds.add(kv_b[0][0])
        first_back = next((nm for nm, _ in rest if is_back_rest(nm)), None)
        if first_back is not None:
            bounds.add(first_back)
            i0 = [nm for nm, _ in rest].index(first_back)
            assert all(is_back_rest(nm) for nm, _ in rest[i0:]), "blocks.* / final_layer.* must close the parameter order"
        after_kv_b = rest[0][0] if rest else None
        if kv_b and after_kv_b is not None:
            bounds.add(after_kv_b)
        off = 0
        ra = self.RANGE_ALIGN
        for name, shape in self.order:
            n = _numel(shape)
            if name in bounds:
                off = (off + ra - 1) // ra * ra
            assert off % self.ALIGN == 0
            self.slots[name] = (off, tuple(shape))
            off += (n + self.ALIGN - 1) // self.ALIGN * self.ALIGN
        self.total = (off + ra - 1) // ra * ra
        self.back_start = self.slots[first_back][0] if first_back is not None else self.total
        self.kv_back = (self.slots[kv_b[0][0]][0], self.slots[after_kv_b][0]) if (kv_b and after_kv_b) else None

        # adaLN stack
        self.ada_rows = sum(s[1][0] for s in ada_w)
        self.ada_offset: Dict[str, int] = {}  # block name (or "final_layer") -> first row in the stack
        r = 0
        for name, shape in ada_w:
            self.ada_offset[name[: -len(".adaLN_modulation.1.weight")]] = r
            r += shape[0]
        self.ada_w_offset = self.slots[ada_w[0][0]][0]
        self.ada_b_offset = self.slots[ada_b[0][0]][0]
        # contiguity of the stacks (no padding holes)
        assert self.slots[ada_w[-1][0]][0] + _numel(ada_w[-1][1]) - self.ada_w_offset == self.ada_rows * cfg.dim
        assert self.slots[ada_b[-1][0]][0] + _numel(ada_b[-1][1]) - self.ada_b_offset == self.ada_rows

        self.groups: Dict[str, MatGroup] = {}
        self.groups["ada"] = MatGroup("ada", self.ada_w_offset, 1, self.ada_rows, cfg.dim)
        for gname, lst in (("kv.patch_mixer", kv_m), ("kv.blocks", kv_b)):
            if not lst:
                continue
            o0 = self.slots[lst[0][0]][0]
            rows = sum(s[1][0] for s in lst)
            cols = lst[0][1][1]
            assert all(s[1][1] == cols for s in lst)
            assert self.slots[lst[-1][0]][0] + _numel(lst[-1][1]) - o0 == rows * cols, "kv stack must be contiguous"
            self.groups[gname] = MatGroup(gname, o0, 1, rows, cols)
        for name, shape in rest:
            if len(shape) < 2:
                continue
            o = self.slots[name][0]
            if name.endswith("mlp.gate.weight"):
                continue  # expert gate stays fp32 (read by md_moe_gate_fwd directly)
            if name.endswith("cross_attn.kv_linear.weight"):
                continue  # part of a kv.* stack
            if len(shape) == 3:  # expert banks [E, in, out]
                self.groups[name] = MatGroup(name, o, shape[0], shape[1], shape[2])
            elif len(shape) == 4:  # patch-embed conv as [D, C*p*p]; its input is data: no dgrad
                self.groups[name] = MatGroup(name, o, 1, shape[0], _numel(shape[1:]), need_t=False)
            elif name.endswith("mlp.w2.weight") and name[: -len("w2.weight")] + "w1.weight" in self.slots:
                continue  # covered by the w12 stack below
            elif name.endswith("mlp.w1.weight"):
                o2 = self.slots[name[: -len("w1.weight")] + "w2.weight"][0]
                assert o2 == o + _numel(shape), "w1/w2 must be adjacent"
                self.groups[name[: -len("w1.weight")] + "w12"] = MatGroup(name[: -len("w1.weight")] + "w12", o, 1,
                                                                         2 * shape[0], shape[1])
            else:
                need_t = name != "y_embedder.y_proj.fc1.weight"  # input is data: no dgrad
                self.groups[name] = MatGroup(name, o, 1, shape[0], shape[1], need_t=need_t)

        # use_bias=True: the fp32 bias vector of each stacked GEMM, group name -> (offset, length).  A w12 stack's is
        # [b1 | b2] in the parameters' own order; a kv.* stack's is every block's [2D] kv_linear bias in block order.
        self.bias: Dict[str, Tuple[int, int]] = {}
        for gname, lst in (("kv.patch_mixer", kvb_m), ("kv.blocks", kvb_b)):
            if lst:
                o0, n = self.slots[lst[0][0]][0], sum(s[1][0] for s in lst)
                assert self.slots[lst[-1][0]][0] + lst[-1][1][0] - o0 == n, "kv bias stack must be contiguous"
                self.bias[gname] = (o0, n)
        for gname, g in self.groups.items():
            pre = gname[: -len("w12")]
            if gname.endswith(".w12") and pre + "w1.bias" in self.slots:
                o1, f = self.slots[pre + "w1.bias"][0], g.rows // 2
                assert self.slots[pre + "w2.bias"][0] == o1 + f, "b1 / b2 must be adjacent"
                self.bias[gname] = (o1, 2 * f)


class ParamStore:
    """Device buffers for one DiT: fp32 master + grad, bf16 copies, views."""

    def __init__(self, layout: ParamLayout, device, lowp_dtype=torch.bfloat16):
        self.layout = layout
        self.device = torch.device(device)
        n = layout.total
        self.flat = torch.zeros(n, dtype=torch.float32, device=self.device)
        self.grad = torch.zeros(n, dtype=torch.float32, device=self.device)
        self.wb = torch.zeros(n, dtype=lowp_dtype, device=self.device)
        self.wbt = torch.zeros(n, dtype=lowp_dtype, device=self.device)
        # fused SwiGLU (MD_EPI_SWIGLU, bf16 mode): the bf16 copies of every w1 | w2 stack interleave the two halves in blocks
        # of 32 rows, so that the GEMM epilogue finds u1 and u2 of a column in the same lane; the fp32 master weights and
        # gradients keep the parameters' own order.  group name -> f (0 / absent: plain order)
        self.interleave: Dict[str, int] = {}
        if lowp_dtype == torch.bfloat16 and os.environ.get("MD_FUSE_SWIGLU", "1") != "0":
            for g in layout.groups.values():
                if g.name.endswith(".w12") and g.batch == 1 and (g.rows // 2) % 32 == 0 and g.cols % 16 == 0:
                    self.interleave[g.name] = g.rows // 2
        self._cast_tables: Dict[str, object] = {}
        self._copies_version: Dict[str, object] = {}
        self.param_ready: Dict[str, object] = {}  # part -> CUDA event of a pending parameter all-gather
        self.p: Dict[str, torch.Tensor] = {}  # fp32 views (reference shapes)
        self.g: Dict[str, torch.Tensor] = {}  # grad views
        for name, (off, shape) in layout.slots.items():
            k = _numel(shape)
            self.p[name] = self.flat[off:off + k].view(shape)
            self.g[name] = self.grad[off:off + k].view(shape)
        self.ada_bias = self.flat[layout.ada_b_offset: layout.ada_b_offset + layout.ada_rows]
        self.g_ada_bias = self.grad[layout.ada_b_offset: layout.ada_b_offset + layout.ada_rows]

    # group views ---------------------------------------------------------------------------
    def _gview(self, buf, g: MatGroup, transposed=False):
        t = buf[g.offset: g.offset + g.numel]
        if transposed:
            return t.view(g.batch, g.cols, g.rows) if g.batch > 1 else t.view(g.cols, g.rows)
        return t.view(g.batch, g.rows, g.cols) if g.batch > 1 else t.view(g.rows, g.cols)

    def W(self, name: str) -> torch.Tensor:
        """bf16 copy in the parameter's own layout ([rows, cols] or [E, rows, cols])."""
        return self._gview(self.wb, self.layout.groups[name])

    def WT(self, name: str) -> torch.Tensor:
        """bf16 transposed copy ([cols, rows] or [E, cols, rows])."""
        g = self.layout.groups[name]
        assert g.need_t, name
        return self._gview(self.wbt, g, transposed=True)

    def G(self, name: str) -> torch.Tensor:
        """fp32 gradient view of a group in its own layout."""
        return self._gview(self.grad, self.layout.groups[name])

    def _bias_slice(self, buf, key: str):
        hit = self.layout.bias.get(key)
        if hit is not None:
            return buf[hit[0]: hit[0] + hit[1]]
        if key.endswith(".weight"):
            hit = self.layout.slots.get(key[: -len("weight")] + "bias")
            if hit is not None:
                return buf[hit[0]: hit[0] + hit[1][0]]
        return None

    def bias(self, key: str):
        """fp32 bias of a GEMM group (a w12 or kv.* stack) or of a single Linear given by its weight name; None when the
        layer has no bias."""
        return self._bias_slice(self.flat, key)

    def gbias(self, key: str):
        """Gradient view matching bias(key)."""
        return self._bias_slice(self.grad, key)

    def is_back(self, offset: int) -> bool:
        """True for tensors of the "back" exchange ranges (backbone blocks, final layer, stacked backbone K/V)."""
        lay = self.layout
        return offset >= lay.back_start or (lay.kv_back is not None and lay.kv_back[0] <= offset < lay.kv_back[1])

    def _cast_table(self, part: str):
        """md_cast_desc rows (one per matrix; expert banks contribute one row per expert) of the groups of `part`, on the
        device, built once: the bf16 copies of a whole exchange range are one launch."""
        hit = self._cast_tables.get(part)
        if hit is not None:
            return hit
        rows, t = [], 0
        for g in self.layout.groups.values():
            if self.is_back(g.offset) != (part == "back"):
                continue
            tx, ty = (g.cols + 63) // 64, (g.rows + 63) // 64
            for b in range(g.batch):
                rows.append([g.offset + b * g.rows * g.cols, g.rows, g.cols, self.interleave.get(g.name, 0), int(g.need_t),
                             t, tx, 0])
                t += tx * ty
        desc = torch.tensor(rows, dtype=torch.int64, device=self.device).reshape(-1, 8).contiguous()
        self._cast_tables[part] = (desc, t)
        return desc, t

    def refresh_copies(self, ops, token=None, force=False, part=None) -> bool:
        """Re-derive the bf16 operand copies if the master weights changed since the last call.
        `token` is any value that changes whenever a parameter is written (models/dit.py sums the
        parameters' autograd version counters, which every in-place optimizer / load_state_dict update bumps).
        `part` = "front" | "back" | None (both): the forward refreshes the front part (stem, patch mixer) when it starts
        and the back part (backbone, final layer) right before the backbone, so that a sharded optimizer's parameter
        all-gather of the back range (train_step.GradReducer.gather_params) overlaps the patch-mixer forward.  Each part
        first makes the compute stream wait for that range's all-gather event, if one is pending."""
        v = token if token is not None else self.flat._version
        done = False
        for pt in (("front", "back") if part is None else (part,)):
            ev = self.param_ready.pop(pt, None)
            if ev is not None:
                torch.cuda.current_stream(self.device).wait_event(ev)
            if not force and self._copies_version.get(pt) == v:
                continue
            desc, tiles = self._cast_table(pt)
            ops.cast_transpose_multi(self.flat, self.wb, self.wbt, desc, tiles)
            self._copies_version[pt] = v
            done = True
        return done
