# -*- coding: utf-8 -*-
"""Host-side logic that needs no GPU: generation-mode selection, kwargs validation, bench sharding over a
world_size-2 gloo group (the N>1 path is independent replicas + one weight broadcast)."""
import json
import os
import subprocess
import sys
import textwrap

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _model():
    from transformers import LlamaConfig
    from painlessinferenceacceleration_b200.models.llama.modeling_llama import LlamaForCausalLM
    cfg = LlamaConfig(vocab_size=64, hidden_size=256, intermediate_size=256, num_hidden_layers=1,
                      num_attention_heads=2, num_key_value_heads=2)
    return LlamaForCausalLM(cfg, device='cpu')


def test_generation_mode_selection():
    from painlessinferenceacceleration_b200.common.lookahead_generation_utils import GenerationMode
    m = _model()
    g = m._get_generation_mode
    assert g(False, True, {'use_lookahead': True}) == GenerationMode.LOOKAHEAD_GENERATION          # reference :72-77
    assert g(False, True, {'use_lookahead': True, 'decoding_length': 1}) == GenerationMode.GREEDY_SEARCH
    assert g(False, True, {'use_lookahead': True, 'branch_length': 0}) == GenerationMode.GREEDY_SEARCH
    assert g(False, False, {'use_lookahead': True}) == GenerationMode.GREEDY_SEARCH
    assert g(False, True, {}) == GenerationMode.GREEDY_SEARCH


def test_unknown_generate_kwargs_raise_like_the_reference():
    m = _model()
    with pytest.raises(ValueError):
        m.generate(input_ids=torch.zeros((1, 4), dtype=torch.long), not_a_real_kwarg=1)  # reference :1309-1317


def test_hf_checkpoint_roundtrip(tmp_path):
    """from_pretrained reads an HF checkpoint directory unchanged (module tree / parameter names are HF's)"""
    from transformers import LlamaConfig, LlamaForCausalLM as HF
    from painlessinferenceacceleration_b200.models.llama.modeling_llama import LlamaForCausalLM
    cfg = LlamaConfig(vocab_size=64, hidden_size=256, intermediate_size=256, num_hidden_layers=2,
                      num_attention_heads=2, num_key_value_heads=2)
    torch.manual_seed(0)
    hf = HF(cfg).to(torch.bfloat16)
    hf.save_pretrained(tmp_path)
    ours = LlamaForCausalLM.from_pretrained(str(tmp_path), device='cpu')
    sd = hf.state_dict()
    for k, v in ours.state_dict().items():
        assert torch.equal(v, sd[k]), k
    ours.fuse()
    w = ours.model.layers[1].self_attn.qkv_weight
    assert torch.equal(w[:256], sd['model.layers.1.self_attn.q_proj.weight'])
    assert ours.model.layers[1].self_attn.k_proj.weight.data_ptr() == w[256:].data_ptr()


def test_phrase_bank_prompts_are_seeded():
    sys.path.insert(0, ROOT)
    import bench
    a = bench.phrase_bank_prompts(3, 32000)
    b = bench.phrase_bank_prompts(3, 32000)
    assert a == b and all(len(p) == 256 and min(p) >= 3 and max(p) < 32000 for p in a)


def test_replica_work_and_aggregation_gloo_world2(tmp_path):
    """N>1 path on CPU: 2 ranks over gloo take their timed requests from bench.timed_requests (identical work per
    replica: the aggregate then scales with the hardware, not with which shard accepts longer drafts), broadcast
    'weights' from rank 0 and aggregate tokens with SUM / time with MAX - no data-path collective."""
    script = tmp_path / 'w.py'
    script.write_text(textwrap.dedent('''
        import os, sys, torch, torch.distributed as dist
        sys.path.insert(0, %r)
        import bench
        dist.init_process_group('gloo')
        rank, world = dist.get_rank(), dist.get_world_size()
        K = 3
        mine = bench.timed_requests(K, rank)
        w = torch.full((8,), float(rank + 1))
        dist.broadcast(w, src=0)
        assert float(w.sum()) == 8.0
        ms = [torch.zeros((1,)) for _ in range(world)]
        dist.all_gather(ms, torch.tensor([10.0 + rank]))
        agg = torch.tensor([float(len(mine) * 256)]); dist.all_reduce(agg)
        idx = torch.tensor(mine); gathered = [torch.zeros_like(idx) for _ in range(world)]
        dist.all_gather(gathered, idx)
        assert all(g.tolist() == mine for g in gathered) and max(mine) < 64, gathered   # identical, inside the timed set
        if rank == 0:
            print('OK', max(float(t) for t in ms), float(agg))
        dist.destroy_process_group()
    ''' % ROOT))
    env = dict(os.environ, MASTER_ADDR='127.0.0.1', MASTER_PORT='29571')
    out = subprocess.run([sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node=2',
                          '--master-addr', '127.0.0.1', '--master-port', '29571', str(script)], env=env,
                         capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr[-2000:]
    assert 'OK 11.0 1536.0' in out.stdout


def test_reference_arm_under_torchrun_prints_one_line_from_rank0():
    """bench.py --impl reference under the driver's N>1 launch: rank 0 alone runs the CPU path (oracle loop + oracle
    trie on the tiny shape here) and prints the one JSON line with its cpu_baseline / e2e objects; the other rank
    exits 0 without output"""
    import json
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node=2',
                          '--master-addr', '127.0.0.1', '--master-port', '29573', os.path.join(root, 'bench.py'),
                          '--impl', 'reference', '--model', 'tiny', '--gpus', '2', '--steps', '2', '--warmup', '1'],
                         capture_output=True, text=True, timeout=600, cwd=root)
    assert out.returncode == 0, out.stderr[-2000:]
    lines = [l for l in out.stdout.splitlines() if l.startswith('{')]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d['impl'] == 'reference' and d['n_gpus'] == 2 and d['steps'] == 2 and d['unit'] == 'tokens/s'
    assert d['value'] > 0 and d['e2e']['value'] == d['value'] and d['e2e']['h2d_bytes_per_step'] == 0
    assert d['cpu_baseline']['kind'] == 'port' and d['cpu_baseline']['cores'] >= 1
    assert d['mean_accepted_len_per_step'] >= 1.0


def test_bench_helpers_traffic_lookup_and_synthetic_weights(tmp_path):
    """bench.py host helpers: roofline.traffic comes from the newest ncu summary whose capture name and kernel match;
    the synthetic weights are a pure function of (name, index) - the GPU arm and the CPU arms build the same model -
    and make greedy decoding follow the successor chain when the embedding dominates"""
    import bench
    (tmp_path / 'r01_traffic.json').write_text(json.dumps({'prof_attn_short_r1:k_tree_attn': 5e6}))
    (tmp_path / 'r02_traffic.json').write_text(json.dumps({'prof_attn_short_r2:k_tree_attn': 9e6,
                                                           'prof_gemm_ws_r2:k_gemm_ws<4>': 1.8e8}))
    t = bench.ncu_traffic('prof_attn_short', 'k_tree_attn', str(tmp_path))
    assert t is not None and 1e6 < t < 1e9 and t == 9e6
    assert bench.ncu_traffic('no_such_capture', 'k_tree_attn', str(tmp_path)) is None
    hbm, tf, src = bench.peaks()
    assert hbm > 1000 and tf > 100 and src in ('measured', 'fallback')
    a = bench.hashed_normal_(torch.empty((3, 1 << 16), dtype=torch.bfloat16), 77, 0.02)
    b = bench.hashed_normal_(torch.empty((3, 1 << 16), dtype=torch.bfloat16), 77, 0.02)
    c = bench.hashed_normal_(torch.empty((3, 1 << 16), dtype=torch.bfloat16), 78, 0.02)
    assert torch.equal(a, b) and not torch.equal(a, c)
    assert abs(a.float().std().item() - 0.02) < 1e-3 and abs(a.float().mean().item()) < 1e-3
    succ = bench.successor_map(32000)
    assert succ.shape == (32000,) and int(succ[3:].min()) >= 3 and int(succ.max()) < 32000
    assert len(set(succ[3:].tolist())) < 31997 * 0.7          # not injective: chains merge
    assert bench.metric_name('mistral-7b').startswith('accepted tokens/sec @ Mistral-7B 64-draft/8-branch')
    torch.set_num_threads(4)
    m = bench.build_cpu_model('tiny')
    cfg, _ = bench.make_config('tiny')
    bench.synth_fill(m, cfg, embed_std=1.0)   # 4 tiny layers: the chain dominates at std 1 (the 7B shape needs ~5.5)
    from oracle.loop import greedy_generate
    p = torch.tensor([bench.phrase_bank_prompts(1, cfg.vocab_size)[0][:32]])
    seq = greedy_generate(m, p, max_new_tokens=12)['sequences'][0].tolist()
    assert all(int(succ[x]) == y for x, y in zip(seq[31:-1], seq[32:]))


def test_weight_layout_helpers_are_permutations():
    """ops.tile_weight ([N, K] -> [N/128, K/64, 128, 64] blocks, the unit k_gemm_ws' TMA box moves) and
    ops.interleave_gate_up (64 gate rows + the 64 up rows of the same columns per 128-row tile) only permute rows /
    blocks: every element survives exactly once (CPU tensors, no library call)"""
    from painlessinferenceacceleration_b200.common import ops
    w = torch.arange(256 * 192, dtype=torch.float32).view(256, 192).to(torch.bfloat16)
    t = ops.tile_weight(w)
    assert t.shape == (2, 3, 128, 64) and t.pia_shape == (256, 192) and t.is_contiguous()
    assert torch.equal(t.permute(0, 2, 1, 3).reshape(256, 192), w)
    assert torch.equal(t[1, 2], w[128:256, 128:192])
    gu = torch.arange(512 * 64, dtype=torch.float32).view(512, 64)
    il = ops.interleave_gate_up(gu)
    assert il.shape == gu.shape
    assert torch.equal(il[0:64], gu[0:64]) and torch.equal(il[64:128], gu[256:320])
    assert torch.equal(il[128:192], gu[64:128]) and torch.equal(il[192:256], gu[320:384])
    assert torch.equal(il.sort(0).values, gu.sort(0).values)
