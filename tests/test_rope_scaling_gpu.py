"""Scaled RoPE (Llama-3.1 / 3.2 ``llama3`` frequencies) on the GPU: the QKV epilogue reading a frequency table against
an fp64 rotation with the same fp32 table, whole pieces against the torch oracle, and EOS lists in the GPU engine."""
import dataclasses
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_gemm_ref_gpu import (EPI_QKV_ROPE, Operands, Run, _bits, _report, check_run, gemm_ref64,  # noqa: E402
                               qkv_rows, run_twice)

from bee2bee_b200.engine.core import Engine, SamplingParams  # noqa: E402
from bee2bee_b200.engine.runner import GpuRunner, SeqInit  # noqa: E402
from bee2bee_b200.models.config import resolve_config, rope_inv_freq  # noqa: E402
from bee2bee_b200.models.torch_ref import TorchPiece  # noqa: E402
from bee2bee_b200.models.weights import init_random, save_hf_dir  # noqa: E402


# --------------------------------------------------------------------------- QKV epilogue + table vs fp64
class TableRun(Run):
    """A QKV + RoPE call that passes ``rope_freq``; its reference rotates by pos * table[j] in fp64."""

    def __init__(self, op, bn, splitk, heads, table, seed):
        super().__init__(op, EPI_QKV_ROPE, bn, 0, splitk, dict(bias=True, theta=500000.0, heads=heads, rstd=False,
                                                               out2=False), seed)
        self.table = table.cuda()

    def launch(self, bufs, **extra):
        return super().launch(bufs, **{"rope_freq": self.table, **extra})

    def ref(self, **mut):
        q = self.qkv
        res = gemm_ref64(self.op, EPI_QKV_ROPE, bias=self.bias, qkv=dict(q, theta=0.0))     # unrotated
        n_out = self.op.n_out
        sect, _, j = qkv_rows(q["n_q"], q["n_kv"], q["hd"], "cuda")
        a = res["pre"] + self.bias.double()[None, :]
        th = q["positions"].double()[:, None] * self.table.double()[j][None, :]
        idx = torch.arange(n_out, device="cuda")
        partner = a[:, idx ^ 1]
        odd = (idx % 2 == 1)[None, :]
        rot = (sect < 2)[None, :]
        o = torch.where(rot, torch.where(odd, a * th.cos() + partner * th.sin(), a * th.cos() - partner * th.sin()), a)
        q_dim, kv_dim = q["n_q"] * q["hd"], q["n_kv"] * q["hd"]
        qs = torch.ones(n_out, dtype=torch.float64, device="cuda")
        qs[:q_dim] = q["q_scale"]
        o = o * qs
        res["fn"] = torch.where(rot, torch.sqrt(a * a + partner * partner), a * 0) * qs
        res["theta"] = torch.where(rot, th, th * 0)
        res["q"], res["k"], res["v"] = o[:, :q_dim], o[:, q_dim:q_dim + kv_dim], o[:, q_dim + kv_dim:]
        res["out"] = o
        return res


TABLE_CASES = [  # (qm, m, bn, splitk, model whose table and head shape are used)
    (0, 24, 16, 4, "llama-3.1-8b"), (0, 150, 128, 1, "llama-3.2-1b"), (0, 300, 256, 2, "llama-3.1-8b"),
    (1, 24, 32, 2, "llama-3.2-1b"), (1, 150, 128, 2, "llama-3.1-8b"),
    (2, 24, 32, 2, "llama-3.1-8b"), (2, 150, 128, 1, "llama-3.2-1b"),
]


@pytest.mark.parametrize("qm,m,bn,splitk,model", TABLE_CASES)
def test_qkv_rope_table_matches_ref64(qm, m, bn, splitk, model):
    """positions up to 131071 on exact pre-activations: outputs within the RoPE angle error of the fp64 rotation by the
    same fp32 table, sentinels and guard rows intact, identical bytes twice.  A null table gives the bytes of a call
    without the argument, and those differ from the table's (the table is what the kernel read)."""
    cfg = resolve_config(model)
    heads = (cfg.head_dim, 4 if cfg.head_dim == 64 else 2, 2 if cfg.head_dim == 64 else 1)
    n_out = (heads[1] + 2 * heads[2]) * heads[0]
    seed = 1000 * qm + m + bn + splitk
    op = Operands(qm, m, 1024, n_out, bn, seed, "cuda", rstd=qm == 1)
    run = TableRun(op, bn, splitk, heads, rope_inv_freq(cfg), seed + 1)
    bufs = run_twice(run, f"table q{qm} m{m}")
    check_run(run, bufs, f"rope table {model} q{qm} m{m} bn{bn} splitk{splitk}")
    none = Run.launch(run, run.fresh(), rope_freq=None)
    absent = Run.launch(run, run.fresh())
    for name in absent:
        assert torch.equal(_bits(none[name]), _bits(absent[name])), name
    assert not torch.equal(_bits(bufs["q"]), _bits(absent["q"]))
    _report()


def test_rope_freq_refused():
    """a table of the wrong length, dtype, device or layout is refused before the launch"""
    cfg = resolve_config("llama-3.2-1b")
    op = Operands(0, 8, 1024, 512, 16, 5, "cuda")
    run = TableRun(op, 16, 1, (64, 4, 2), rope_inv_freq(cfg), 6)
    good = run.table
    for bad in (good[:-1], good.double(), good.cpu(), good.repeat(2)[::2], good.to(torch.bfloat16)):
        with pytest.raises(RuntimeError, match="rope_freq"):
            Run.launch(run, run.fresh(), rope_freq=bad)


# --------------------------------------------------------------------------- whole pieces vs the oracle
def _sharp_dir(tmp_path, cfg, qk_gain=4.0):
    """random tiny weights with q / k rows scaled so attention is peaked: RoPE frequencies then move the logits well
    beyond the kernels' rounding (with std 0.02 projections attention is nearly uniform)"""
    t = init_random(cfg, range(cfg.n_layers), True, True, seed=0)
    for k in t:
        if k.endswith((".wq", ".wk")):
            t[k] = t[k] * qk_gain
    d = str(tmp_path / cfg.name)
    save_hf_dir(d, cfg, t, dtype=torch.bfloat16)
    return d


def _oracles(cfg, model_dir):
    from bee2bee_b200.models.weights import load_hf_dir
    t = load_hf_dir(model_dir, cfg, range(cfg.n_layers), True, True, device="cuda", dtype=torch.float32)
    plain = dataclasses.replace(cfg, rope_scaling=None)
    return (TorchPiece(cfg, range(cfg.n_layers), True, True, t), TorchPiece(plain, range(cfg.n_layers), True, True, t))


def _rel_err(a, b):
    return ((a.float() - b.float()).abs().max() / b.float().abs().max().clamp_min(1e-6)).item()


def _decode_against_oracles(cfg, model_dir, quant, prompts, steps=5):
    """chunked prefill of ``prompts`` then greedy decode steps; per step the GPU logits and the logits of the scaled and
    the unscaled oracle fed the same tokens.  Returns [(got, scaled, unscaled)]."""
    runner = GpuRunner(cfg, model_dir, 0, 1, torch.device("cuda:0"), max_batch=4, groups=1, max_seq_len=512,
                       max_prefill_tokens=128, seed=0, use_graphs=True, quant=quant)
    scaled, unscaled = _oracles(cfg, model_dir)
    V = cfg.vocab_size
    n = len(prompts)
    seqs = [SeqInit(slot=i, prompt=p, pages=list(range(1 + 8 * i, 9 + 8 * i)), temperature=0.0, top_p=1.0,
                    repetition_penalty=1.0, seed=i) for i, p in enumerate(prompts)]
    runner.prefill(seqs)
    runner.sync()
    caches = [[o.new_cache() for _ in seqs] for o in (scaled, unscaled)]
    with torch.no_grad():
        for o, cs in zip((scaled, unscaled), caches):
            for s, c in zip(seqs, cs):
                o.forward(torch.tensor([s.prompt], device="cuda"), torch.arange(len(s.prompt), device="cuda")[None], c)
    out = []
    for step in range(steps):
        fed = runner.tokens[:n].tolist()
        runner.decode(1)
        runner.sync()
        got = runner.piece.logits[:n, :V].clone()
        with torch.no_grad():
            for b in range(n):
                ids = torch.tensor([[fed[b]]], device="cuda")
                pos = torch.tensor([[len(seqs[b].prompt) + step]], device="cuda")
                refs = [o.forward(ids, pos, cs[b])[0, -1] for o, cs in zip((scaled, unscaled), caches)]
                out.append((got[b], refs[0], refs[1]))
    runner.close()
    return out


@pytest.mark.parametrize("quant", ["bf16", "mxfp8"])
def test_piece_with_scaled_rope_matches_oracle(quant, tmp_path):
    """tiny-llama31 (original context 64) with 150-300 token prompts: bf16 within test_piece_matches_oracle's 6e-2, MX
    fp8 within test_piece_fp8_close_to_oracle's 0.2 / cosine 0.98, and the GPU logits several times closer to the
    scaled oracle than to the same model with plain RoPE"""
    cfg = resolve_config("tiny-llama31")
    d = _sharp_dir(tmp_path, cfg)
    cfg = resolve_config(d)
    assert cfg.rope_scaling == resolve_config("tiny-llama31").rope_scaling
    V = cfg.vocab_size
    prompts = [[(7 * i + 3) % V for i in range(150)], [(5 * i + 11) % V for i in range(300)],
               [(13 * i + 1) % V for i in range(211)]]
    res = _decode_against_oracles(cfg, d, quant, prompts)
    d_scaled = torch.stack([(g - s).norm() for g, s, _ in res]).norm().item()
    d_plain = torch.stack([(g - u).norm() for g, _, u in res]).norm().item()
    for i, (g, s, _) in enumerate(res):
        err = _rel_err(g, s)
        if quant == "bf16":
            assert err < 6e-2, f"step/seq {i}: rel err {err}"
        else:
            assert err < 0.2, f"step/seq {i}: rel err {err}"
            cos = torch.nn.functional.cosine_similarity(g.float(), s.float(), dim=0).item()
            assert cos > 0.98, cos
    # measured on CPU stand-ins of the rounding: about 45x (bf16) and 4x (MX fp8)
    need = 8.0 if quant == "bf16" else 2.0
    assert d_plain > need * d_scaled, (d_plain, d_scaled)


@pytest.mark.parametrize("shape", ["llama-3.2-1b", "llama-3.2-3b"])
def test_llama32_shapes_match_oracle(shape, tmp_path):
    """two layers of Llama-3.2-1B (head_dim 64, tensor-core attention) and Llama-3.2-3B (GQA 3, CUDA-core attention)
    with a 512-token vocabulary, bf16, against the oracle"""
    from bee2bee_b200 import ops
    full = resolve_config(shape)
    cfg = dataclasses.replace(full, name=f"tiny-{shape}", n_layers=2, vocab_size=512, eos_token_id=1, bos_token_id=0,
                              eos_token_ids=())
    g = cfg.n_heads // cfg.n_kv_heads
    assert (cfg.head_dim, g) == ((64, 4) if shape == "llama-3.2-1b" else (128, 3))
    if g == 3:
        assert not ops.native().attention_uses_tc(128, cfg.n_heads, cfg.n_kv_heads, cfg.head_dim)
    d = _sharp_dir(tmp_path, cfg, qk_gain=1.0)
    cfg = resolve_config(d)
    V = cfg.vocab_size
    prompts = [[(7 * i + 3) % V for i in range(150)], [(5 * i + 11) % V for i in range(70)], [4, 9, 2]]
    res = _decode_against_oracles(cfg, d, "bf16", prompts, steps=4)
    for i, (got, ref, _) in enumerate(res):
        err = _rel_err(got, ref)
        assert err < 6e-2, f"{shape} step/seq {i}: rel err {err}"


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
def test_two_gpu_scaled_rope_matches_single_gpu():
    from test_multigpu import _run
    ref = _run(1, "tiny-llama31", 2, 4, 0)
    got = _run(2, "tiny-llama31", 2, 4, 29631)
    assert got == ref


# --------------------------------------------------------------------------- EOS lists on the GPU engine
def test_gpu_engine_stops_on_a_later_eos_id():
    sp = SamplingParams(max_new_tokens=12, temperature=0.0, ignore_eos=True)
    prompt = [(7 * i + 3) % 512 for i in range(80)]
    eng = Engine("tiny-llama31", device="cuda:0", max_batch=2, max_seq_len=256, decode_burst=4)
    free = eng.generate([prompt], sp)[0]
    eng.close()
    stop = free[5]
    first = free.index(stop)
    base = resolve_config("tiny-llama31")
    other = next(t for t in range(2, 512) if t not in free)
    cfg = dataclasses.replace(base, eos_token_id=other, eos_token_ids=(other, stop))
    eng = Engine("tiny-llama31", cfg=cfg, device="cuda:0", max_batch=2, max_seq_len=256, decode_burst=4)
    req = eng.submit(prompt, SamplingParams(max_new_tokens=12, temperature=0.0))
    eng.start()
    req.wait(timeout=120)
    eng.stop()
    eng.close()
    assert req.out_ids == free[:first + 1] and req.finish_reason == "stop"
