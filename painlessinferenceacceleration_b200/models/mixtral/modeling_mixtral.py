# -*- coding: utf-8 -*-
"""Mixtral with the lookahead patch (reference: models/mixtral/modeling_mixtral.py, patch :1032-1036, attention
:302-381, MixtralSparseMoeBlock :692-759, expert MLP :668-683).

Attention / norms / RoPE are the Llama-family kernels (GQA packed into the UMMA tile).  The MoE block: at n = 64
draft nodes with top-2 of 8 routing practically every expert is hit, so the verify step reads all expert weights
either way (SURVEY.md 8d: >= 90 GB per step); the block therefore evaluates every expert on all n rows with
static-shape GEMMs (CUDA-graph friendly, no host-side routing) and combines with the routing weights, zero for
unselected experts.  Rounding follows the reference: fp32 softmax -> top-k -> renormalise -> cast to bf16 (:723-727);
per token the two selected expert outputs are scaled in bf16 and accumulated in expert-index order, exactly what
`index_add_` into a zero tensor produces (:729-757).  An expert whose bf16 weight for a token is 0 is skipped for that
token rather than added as `ye * 0`: the reference never evaluates an unselected expert for the token, so an inf or NaN
in that expert's output must not turn the sum into NaN.  For finite outputs the skip changes no bit (the sum starts at
+0, never becomes -0, and adding +-0 leaves it unchanged).  It differs from the reference only for a selected expert
whose weight underflowed to 0 in bf16 and whose output is not finite: the reference's sum is then NaN, ours is not."""
import os
import re

import torch
from torch import nn

from ...common import ops
from ..llama.modeling_llama import (Fp8Linear, Int4Linear, LlamaDecoderLayer, LlamaForCausalLM, LlamaModel,
                                    _gate_up_order, _w4_spec)
from ..mistral.modeling_mistral import warn_sliding_window


class MixtralRouter(nn.Module):
    def __init__(self, cfg, device, dtype):
        super().__init__()
        self.weight = nn.Parameter(torch.empty((cfg.num_local_experts, cfg.hidden_size), device=device, dtype=dtype))


class MixtralExperts(nn.Module):
    def __init__(self, cfg, device, dtype):
        super().__init__()
        E, H, I = cfg.num_local_experts, cfg.hidden_size, cfg.intermediate_size
        self.gate_up_proj = nn.Parameter(torch.empty((E, 2 * I, H), device=device, dtype=dtype))
        self.down_proj = nn.Parameter(torch.empty((E, H, I), device=device, dtype=dtype))


class Int4Stack(Int4Linear):
    """G int4 weights [N, K] (the MoE experts) stacked by rows into one Int4Linear [G * N, K]: code tiles, scale and
    zero-point tables [K / group, G * N] in the int4 GEMM's layout; `shape` is (G, N, K).  `interleaved`: fused gate/up
    weights whose rows (with their scales and zero points) are put in the SiLU*up epilogue's order per weight, so that
    every 128-row tile holds one expert's 64 gate rows and the 64 up rows of the same columns."""

    def __init__(self, u, s, z, group_size, interleaved=False):
        G, N, K = u.shape
        if interleaved:   # per expert: _gate_up_order keeps the leading (expert) dim
            u, s, z = _gate_up_order(u), _gate_up_order(s), _gate_up_order(z)
        super().__init__(*(t.reshape(G * N, t.shape[-1]) for t in (u, s, z)), group_size)
        self.shape = (G, N, K)
        self.interleaved = interleaved

    def codes(self):
        """(u uint8 [G, N, K], s [G, N, K / group], z uint8 [G, N, K / group]) in the checkpoint's row order; [e] is
        expert e's (u, s, z) as Int4Linear.codes gives them"""
        G, N, K = self.shape
        u = ops.untile_weight_w4(self.qweight, K).view(G, N, K)
        s, z = (t.data.t().reshape(G, N, -1) for t in (self.scale, self.zero))
        if self.interleaved:
            u, s, z = (_gate_up_order(t, inverse=True) for t in (u, s, z))
        return u, s.contiguous(), z.contiguous()

    def dequantize(self):
        """the weights the int4 GEMM multiplies with (ops.dequantize_w4 per expert), bf16 [G, N, K]"""
        u, s, z = self.codes()
        return torch.stack([ops.dequantize_w4(u[e], s[e], z[e], self.group_size) for e in range(self.shape[0])])


class MixtralSparseMoeBlock(nn.Module):
    def __init__(self, cfg, device, dtype):
        super().__init__()
        self.top_k = cfg.num_experts_per_tok
        self.num_experts = cfg.num_local_experts
        self.gate = MixtralRouter(cfg, device, dtype)
        self.experts = MixtralExperts(cfg, device, dtype)


class MixtralDecoderLayer(LlamaDecoderLayer):
    def _make_mlp(self, cfg, device, dtype):
        return MixtralSparseMoeBlock(cfg, device, dtype)


class MixtralModel(LlamaModel):
    layer_cls = MixtralDecoderLayer


class MixtralForCausalLM(LlamaForCausalLM):
    model_cls = MixtralModel
    int4_checkpoints = False   # no int4 weight mode for this family
    rmsnorm_rounding = ops.ROUND_TWICE   # weight * hidden_states.to(input_dtype) (mixtral/modeling_mixtral.py:165)

    def _fuse_mlp(self, layer):
        pass  # experts are stored fused ([E, 2I, H]) already

    @classmethod
    def from_pretrained(cls, path, torch_dtype=torch.bfloat16, device=None, quantization=None, **kwargs):
        """as LlamaForCausalLM.from_pretrained; a GPTQ / compressed-tensors int4 checkpoint (config.quantization_config)
        loads through the expert-aware loader below: the attention projections and every expert in int4, the router,
        embeddings, lm_head and norms in bf16"""
        config = cls._pretrained_config(path)
        if not getattr(config, 'quantization_config', None):
            return super().from_pretrained(path, torch_dtype=torch_dtype, device=device, quantization=quantization,
                                           **kwargs)
        spec = cls._w4_moe_spec(config)
        if quantization is not None:
            raise ValueError(f'quantization={quantization!r}: this checkpoint is already quantised '
                             f'({spec["format"]} int4); load it with quantization=None')
        return cls._from_pretrained_w4(path, config, spec, device)

    def rope_tables(self, max_pos):
        warn_sliding_window(self.config, max_pos)  # mixtral/modeling_mixtral.py:1032-1036: no window on the lookahead branch
        return super().rope_tables(max_pos)

    def _convert_checkpoint_keys(self, sd):
        """published Mixtral checkpoints (and the reference, mixtral/modeling_mixtral.py:692-759) name the MoE block
        `block_sparse_moe` with per-expert `experts.N.w1 / w3 / w2` Linear weights; this module tree keeps the experts
        stacked: gate_up_proj[e] = [w1; w3] ([2I, H]), down_proj[e] = w2 ([H, I]), router = `mlp.gate.weight`.  Tensors
        of one layer's experts may arrive in different shards: partial stacks are kept until complete."""
        import re
        out = {}
        pend = self.__dict__.setdefault('_pending_experts', {})
        E = self.config.num_local_experts
        pat = re.compile(r'^(model\.layers\.\d+)\.block_sparse_moe\.experts\.(\d+)\.(w1|w2|w3)\.weight$')
        for k, v in sd.items():
            m = pat.match(k)
            if m:
                pend.setdefault(m.group(1), {})[(int(m.group(2)), m.group(3))] = v
            elif '.block_sparse_moe.gate.weight' in k:
                out[k.replace('.block_sparse_moe.gate.weight', '.mlp.gate.weight')] = v
            else:
                out[k] = v
        for layer in list(pend):
            parts = pend[layer]
            if len(parts) == 3 * E:
                out[layer + '.mlp.experts.gate_up_proj'] = torch.stack(
                    [torch.cat([parts[(e, 'w1')], parts[(e, 'w3')]], dim=0) for e in range(E)], dim=0)
                out[layer + '.mlp.experts.down_proj'] = torch.stack([parts[(e, 'w2')] for e in range(E)], dim=0)
                del pend[layer]
        return out

    def geometry(self):
        g = super().geometry()
        g['n_experts'] = self.config.num_local_experts
        return g

    def _layer_gemm_plans(self, layer, b):
        """decode steps (64-row buffers): all experts' gate_up as ONE k_gemm_ws launch over the stacked [E*2I, H] weight,
        SiLU*up over the [64*E, 2I] view, all experts' down projections as one grouped launch, then the routing-weighted
        sum in expert order.  Dense over experts like the cuBLAS path below: at n = 64 draft rows every expert is hit
        (SURVEY 8d), and the step is bound by the expert weight bytes either way.  PIA_MOE_GEMM=0 keeps cuBLAS."""
        import os
        moe = layer.mlp
        E, two_i, H = moe.experts.gate_up_proj.shape
        inter = two_i // 2
        if os.environ.get('PIA_MOE_GEMM', '1') == '0' or H % 128 or H % 64 or inter % 64 or (E * two_i) % 128:
            return {}
        dev = b.y.device
        if not hasattr(b, 'moe_gu'):
            b.moe_gu = torch.zeros((b.rows, E * two_i), dtype=torch.bfloat16, device=dev)
            b.moe_act = torch.zeros((b.rows, E * inter), dtype=torch.bfloat16, device=dev)
            b.moe_out = torch.zeros((b.rows, H), dtype=torch.bfloat16, device=dev)
            b.moe_dense = torch.zeros((b.rows, E), dtype=torch.bfloat16, device=dev)
        return {'moe_gate_up': ops.Gemm(moe.experts.gate_up_proj.data.view(E * two_i, H), b.y),
                'moe_down': ops.Gemm.grouped(moe.experts.down_proj.data, b.moe_act)}

    # ------------------------------------------------------------------ fp8: the experts as stacked fp8 weights
    # the experts' stacks are quantised once _convert_checkpoint_keys has assembled them
    _fp8_params = ('self_attn.q_proj.weight', 'self_attn.k_proj.weight', 'self_attn.v_proj.weight',
                   'self_attn.o_proj.weight', 'mlp.experts.gate_up_proj', 'mlp.experts.down_proj')

    def _fp8_weight_shapes(self, layer):
        a, ex = layer.self_attn, layer.mlp.experts
        return [('qkv', a.qkv_weight.shape), ('o_proj', a.o_proj.weight.shape),
                ('experts.gate_up_proj', ex.gate_up_proj.shape), ('experts.down_proj', ex.down_proj.shape)]

    def _quantize_mlp(self, layer):
        ex = layer.mlp.experts
        gu = Fp8Linear(ex.gate_up_proj.data, interleaved=True)   # per expert: 64 gate + 64 up rows per tile
        del ex.gate_up_proj
        ex.gate_up_proj = gu
        dn = Fp8Linear(ex.down_proj.data)
        del ex.down_proj
        ex.down_proj = dn

    @staticmethod
    def _moe_bufs(b, E, inter, H):
        """the MoE block's buffers of the fp8 / int4 plans, over every row of the buffer set"""
        if getattr(b, 'moe_act', None) is None or b.moe_act.shape[0] != b.rows:
            dev = b.y.device
            b.moe_act = torch.zeros((b.rows, E * inter), dtype=torch.bfloat16, device=dev)
            b.moe_out = torch.zeros((b.rows, H), dtype=torch.bfloat16, device=dev)
            b.moe_dense = torch.zeros((b.rows, E), dtype=torch.bfloat16, device=dev)

    def _layer_fp8_plans(self, layer, b, n_sm):
        """qkv / o as in Llama; all experts' gate_up as ONE fp8 launch with the SiLU*up epilogue over the stacked
        [E * 2I, H] weight (writes act [rows, E * I]), all experts' down projections as one grouped fp8 launch"""
        plans = self._attn_fp8_plans(layer, b, n_sm)
        ex = layer.mlp.experts
        E, two_i, H = ex.gate_up_proj.shape
        self._moe_bufs(b, E, two_i // 2, H)
        gq = ex.gate_up_proj.qweight
        plans['moe_gate_up_silu'] = ops.Gemm.fp8(gq.view(-1, *gq.shape[2:]), ex.gate_up_proj.scale.view(-1), b.y,
                                                 out=b.moe_act).set_silu()
        plans['moe_down'] = ops.Gemm.grouped_fp8(ex.down_proj.qweight, ex.down_proj.scale, b.moe_act)
        return plans

    # ------------------------------------------------------------------ int4: GPTQ / compressed-tensors experts
    @staticmethod
    def _w4_moe_spec(config):
        """_w4_spec, plus what the MoE block needs: a router (block_sparse_moe.gate) left unquantised by the
        compressed-tensors `ignore` list (literal names or `re:` patterns, matched as compressed-tensors does)"""
        spec = _w4_spec(config)
        q = config.quantization_config
        q = q.to_dict() if hasattr(q, 'to_dict') else dict(q)
        if spec['format'] == 'compressed-tensors':
            ignore = q.get('ignore') or []
            for li in range(config.num_hidden_layers):
                name = f'model.layers.{li}.block_sparse_moe.gate'
                if not any(i == name or (i.startswith('re:') and re.match(i[3:], name)) for i in ignore):
                    raise ValueError(f'quantization_config.ignore={ignore!r} does not hold {name}: a quantised MoE '
                                     'router is not supported (it stays bf16)')
        return spec

    _W4_ATTN = ('q_proj', 'k_proj', 'v_proj', 'o_proj')
    _W4_KEY = re.compile(r'^model\.layers\.(\d+)\.(self_attn\.[qkvo]_proj|block_sparse_moe\.experts\.\d+\.w[123]|'
                         r'block_sparse_moe\.gate)\.(\w+)$')

    def _install_w4_experts(self, layer, experts):
        """the MoE block's experts from [{'w1': (u, s, z, gs), 'w3': ..., 'w2': ...} per expert]: gate/up as one
        interleaved Int4Stack [E * 2I, H] ([w1_e; w3_e] per expert), down as one Int4Stack [E * H, I]"""
        if len({ex[n][3] for ex in experts for n in ('w1', 'w3')}) != 1:
            raise ValueError('the experts\' w1 / w3 have different group sizes: they cannot be fused')
        if len({ex['w2'][3] for ex in experts}) != 1:
            raise ValueError('the experts\' w2 have different group sizes: they cannot be stacked')
        gate_up = [torch.stack([torch.cat([ex['w1'][i], ex['w3'][i]], dim=0) for ex in experts]) for i in range(3)]
        down = [torch.stack([ex['w2'][i] for ex in experts]) for i in range(3)]
        ex = layer.mlp.experts
        del ex.gate_up_proj, ex.down_proj
        ex.gate_up_proj = Int4Stack(*gate_up, experts[0]['w1'][3], interleaved=True)
        del gate_up
        ex.down_proj = Int4Stack(*down, experts[0]['w2'][3])

    @classmethod
    @torch.no_grad()
    def _from_pretrained_w4(cls, path, config, spec, device):
        """As LlamaForCausalLM._from_pretrained_w4, per expert: everything that stays bf16 is allocated up front; the
        packed tensors of a layer's attention projections and experts (block_sparse_moe.experts.{e}.{w1,w3,w2}) wait on
        the host until the layer is complete, in whatever shards and order they arrive, then the layer is unpacked,
        stacked and tiled on the GPU, so no bf16 expert ever exists there."""
        model, own, _, _ = cls._fp8_skeleton(config, device)
        dev = model.model.norm.weight.device
        E = config.num_local_experts
        parts = cls._W4_PARTS[spec['format']]
        need = {'qweight', 'qzeros', 'scales'} if spec['format'] == 'gptq' else \
            {'weight_packed', 'weight_scale', 'weight_shape'} | (set() if spec['sym'] else {'weight_zero_point'})
        projs = [f'self_attn.{n}' for n in cls._W4_ATTN] + \
            [f'block_sparse_moe.experts.{e}.{x}' for e in range(E) for x in ('w1', 'w3', 'w2')]
        pending = {li: {} for li in range(len(model.model.layers))}
        seen = set()

        def finish(li):
            got = pending.pop(li)
            un = lambda p: cls._w4_unpack(spec, {k: v.to(dev) for k, v in got[p].items()}, f'model.layers.{li}.{p}')
            layer = model.model.layers[li]
            model._install_w4_attn(layer, {n: un(f'self_attn.{n}') for n in cls._W4_ATTN})
            model._install_w4_experts(layer, [{x: un(f'block_sparse_moe.experts.{e}.{x}') for x in ('w1', 'w3', 'w2')}
                                              for e in range(E)])

        for sd in cls._shards(path):
            for k, v in sd.items():
                m = cls._W4_KEY.match(k)
                if m and m.group(2) == 'block_sparse_moe.gate':
                    if m.group(3) != 'weight':
                        raise ValueError(f'{k}: a quantised MoE router is not supported (it stays bf16)')
                    k = f'model.layers.{m.group(1)}.mlp.gate.weight'
                elif m and m.group(3) == 'weight':
                    raise ValueError(f'{k}: this int4 checkpoint stores layer {m.group(1)}\'s {m.group(2)} unquantised; '
                                     'a layer must have every projection in int4')
                elif m and m.group(3) in parts:
                    li = int(m.group(1))
                    if li in pending:
                        pending[li].setdefault(m.group(2), {})[m.group(3)] = v
                    continue
                elif k.rpartition('.')[2] in parts and k.startswith(('lm_head.', 'model.embed_tokens.')):
                    what = 'lm_head' if k.startswith('lm_head.') else 'embedding'
                    raise ValueError(f'{k}: a quantised {what} is not supported (it stays bf16)')
                if k in own:
                    own[k].copy_(v.to(torch.bfloat16))
                    seen.add(k)
            # layers are finished at the end of a shard, so that an optional tensor (g_idx) stored after the required
            # ones in the same shard is not missed
            for li in [li for li, got in pending.items() if all(need <= got.get(p, {}).keys() for p in projs)]:
                finish(li)
        if 'lm_head.weight' not in seen and getattr(config, 'tie_word_embeddings', False):
            model.lm_head.weight.copy_(model.model.embed_tokens.weight)
            seen.add('lm_head.weight')
        missing = [k for k in own if k not in seen]
        missing += [f'model.layers.{li}.* ({sorted(got)[:2]})' for li, got in pending.items()]
        if missing:
            raise RuntimeError(f'checkpoint is missing {len(missing)} tensors, e.g. {missing[:4]}')
        model._fused = True
        model._w4 = True
        return model

    @classmethod
    @torch.no_grad()
    def build_w4(cls, config, fill_rest, fill_codes, device=None):
        """An int4 Mixtral without a checkpoint (synthetic weights: the benchmark's and the big tests' 8x7B / 8x22B
        shapes), as LlamaForCausalLM.build_w4: fill_codes(name, (N, K)) returns each projection's (u, s, z, group size)
        on the GPU, one layer at a time, under the checkpoint's names ('model.layers.3.self_attn.q_proj.weight',
        'model.layers.3.block_sparse_moe.experts.5.w1.weight')."""
        model, _, _, _ = cls._fp8_skeleton(config, device)
        fill_rest(model)
        E, H, I = config.num_local_experts, config.hidden_size, config.intermediate_size
        for li, layer in enumerate(model.model.layers):
            a, pre = layer.self_attn, f'model.layers.{li}.'
            model._install_w4_attn(layer, {n: fill_codes(f'{pre}self_attn.{n}.weight',
                                                         tuple(getattr(a, n).weight.shape)) for n in cls._W4_ATTN})
            model._install_w4_experts(layer, [
                {x: fill_codes(f'{pre}block_sparse_moe.experts.{e}.{x}.weight', (H, I) if x == 'w2' else (I, H))
                 for x in ('w1', 'w3', 'w2')} for e in range(E)])
        model._fused = True
        model._w4 = True
        return model

    def _layer_w4_plans(self, layer, b, n_sm):
        """qkv / o as in Llama; all experts' gate_up as ONE int4 launch with the SiLU*up epilogue over the stacked
        [E * 2I, H] weight (writes act [rows, E * I]), all experts' down projections as one grouped int4 launch.  There
        is no cuBLAS path for int4 experts, so PIA_MOE_GEMM=0 is refused."""
        if os.environ.get('PIA_MOE_GEMM', '1') == '0':
            raise ValueError('this model holds int4 experts, which only the int4 GEMM runs: PIA_MOE_GEMM=0 does not '
                             'apply')
        plans = self._attn_w4_plans(layer, b, n_sm)
        gu, dn = layer.mlp.experts.gate_up_proj, layer.mlp.experts.down_proj
        E, two_i, H = gu.shape
        self._moe_bufs(b, E, two_i // 2, H)
        plans['moe_gate_up_silu'] = gu.gemm(b.y, out=b.moe_act).set_silu()
        plans['moe_down'] = ops.Gemm.grouped_w4(dn.qweight, dn.scale, dn.zero, dn.group_size, E, b.moe_act)
        return plans

    def _mlp(self, rt, layer, y, plans=None, b=None):
        moe = layer.mlp
        if plans:
            b = b if b is not None else rt.decode_bufs
            E = moe.num_experts
            inter = moe.experts.down_proj.shape[2]
            ops.moe_router(y, moe.gate.weight, moe.top_k, b.moe_dense)              # :721-727 in one kernel
            if 'moe_gate_up_silu' in plans:                                         # fp8 / int4: all buffer rows
                rows = y.shape[0]
                plans['moe_gate_up_silu'].run(rows, out=b.moe_act)
                ye = plans['moe_down'].run(rows)                                    # [E, rows, H]
                ops.moe_combine(ye, b.moe_dense, b.moe_out)
                return b.moe_out, None
            plans['moe_gate_up'].run(64, out=b.moe_gu)
            ops.silu_mul(b.moe_gu.view(b.rows * E, 2 * inter), b.moe_act.view(b.rows * E, inter))
            ye = plans['moe_down'].run(64)                                          # [E, 64, H]
            ops.moe_combine(ye, b.moe_dense, b.moe_out)
            return b.moe_out, None
        dense = torch.empty((y.shape[0], moe.num_experts), dtype=y.dtype, device=y.device)
        ops.moe_router(y, moe.gate.weight, moe.top_k, dense)                        # :721-727
        out = torch.zeros_like(y)
        inter = moe.experts.down_proj.shape[2]
        act = torch.empty((y.shape[0], inter), dtype=y.dtype, device=y.device)
        for e in range(moe.num_experts):                                            # expert-index order (:734)
            gu = torch.mm(y, moe.experts.gate_up_proj[e].t())
            ops.silu_mul(gu, act)
            ye = torch.mm(act, moe.experts.down_proj[e].t())
            w = dense[:, e:e + 1]                                                   # bf16 scale, bf16 accumulate;
            out += torch.where(w != 0, ye * w, 0.0)                                 # rows that skip e add +0
        return out, None
