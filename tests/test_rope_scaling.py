"""Llama-3.1 / 3.2 / 3.3 checkpoints on CPU: the llama3 RoPE frequency table, config.json parsing in both the legacy
and the transformers >= 5 layout, the torch oracle against transformers' LlamaForCausalLM past the original context,
and generation stopping at every EOS id the config lists."""
import dataclasses
import json
import math

import pytest
import torch

from bee2bee_b200.engine.core import Engine, SamplingParams
from bee2bee_b200.models.config import PRESETS, ModelConfig, resolve_config, rope_inv_freq
from bee2bee_b200.models.torch_ref import TorchPiece
from bee2bee_b200.models.weights import init_random, save_hf_dir

# published config.json of meta-llama/Llama-3.1-8B-Instruct and meta-llama/Llama-3.2-3B
LLAMA31_8B_INSTRUCT = {
    "architectures": ["LlamaForCausalLM"], "attention_bias": False, "attention_dropout": 0.0, "bos_token_id": 128000,
    "eos_token_id": [128001, 128008, 128009], "hidden_act": "silu", "hidden_size": 4096, "initializer_range": 0.02,
    "intermediate_size": 14336, "max_position_embeddings": 131072, "mlp_bias": False, "model_type": "llama",
    "num_attention_heads": 32, "num_hidden_layers": 32, "num_key_value_heads": 8, "pretraining_tp": 1,
    "rms_norm_eps": 1e-05,
    "rope_scaling": {"factor": 8.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0,
                     "original_max_position_embeddings": 8192, "rope_type": "llama3"},
    "rope_theta": 500000.0, "tie_word_embeddings": False, "torch_dtype": "bfloat16", "transformers_version": "4.42.3",
    "use_cache": True, "vocab_size": 128256}
LLAMA32_3B = {
    "architectures": ["LlamaForCausalLM"], "attention_bias": False, "attention_dropout": 0.0, "bos_token_id": 128000,
    "eos_token_id": 128001, "head_dim": 128, "hidden_act": "silu", "hidden_size": 3072, "initializer_range": 0.02,
    "intermediate_size": 8192, "max_position_embeddings": 131072, "mlp_bias": False, "model_type": "llama",
    "num_attention_heads": 24, "num_hidden_layers": 28, "num_key_value_heads": 8, "pretraining_tp": 1,
    "rms_norm_eps": 1e-05,
    "rope_scaling": {"factor": 32.0, "high_freq_factor": 4.0, "low_freq_factor": 1.0,
                     "original_max_position_embeddings": 8192, "rope_type": "llama3"},
    "rope_theta": 500000.0, "tie_word_embeddings": True, "torch_dtype": "bfloat16",
    "transformers_version": "4.45.0.dev0", "use_cache": True, "vocab_size": 128256}


def _as_rope_parameters(d):
    """the same config as transformers >= 5 writes it: theta inside ``rope_parameters``, top-level keys null"""
    out = {k: v for k, v in d.items() if k not in ("rope_scaling", "rope_theta")}
    out["rope_parameters"] = {**d["rope_scaling"], "rope_theta": d["rope_theta"]}
    out["rope_theta"] = None
    out["rope_scaling"] = None
    return out


def _inv_freq64(cfg):
    """the llama3 transform written out in fp64 from its definition"""
    rs = cfg.rope_scaling
    orig, low, high, factor = (rs["original_max_position_embeddings"], rs["low_freq_factor"], rs["high_freq_factor"],
                               rs["factor"])
    out = []
    for j in range(cfg.head_dim // 2):
        f = cfg.rope_theta ** (-2.0 * j / cfg.head_dim)
        wavelen = 2 * math.pi / f
        if wavelen < orig / high:
            out.append(f)
        elif wavelen > orig / low:
            out.append(f / factor)
        else:
            s = (orig / wavelen - low) / (high - low)
            out.append((1 - s) * f / factor + s * f)
    return torch.tensor(out, dtype=torch.float64)


@pytest.mark.parametrize("name", ["llama-3.1-8b", "llama-3.2-1b", "llama-3.2-3b", "tiny-llama31"])
def test_frequency_table(name):
    cfg = resolve_config(name)
    inv = rope_inv_freq(cfg)
    assert inv.dtype == torch.float32 and inv.shape == (cfg.head_dim // 2,) and inv.is_contiguous()
    ref = _inv_freq64(cfg)
    assert torch.allclose(inv.double(), ref, rtol=2e-6, atol=0), (inv.double() / ref - 1).abs().max()
    # the scaling moves a large share of the pairs: at least a third of them run `factor` times slower
    plain = cfg.rope_theta ** (-torch.arange(0, cfg.head_dim, 2, dtype=torch.float64) / cfg.head_dim)
    slow = torch.isclose(ref, plain / cfg.rope_scaling["factor"], rtol=1e-12).sum().item()
    assert slow >= cfg.head_dim // 6, slow
    transformers = pytest.importorskip("transformers")
    from transformers.modeling_rope_utils import ROPE_INIT_FUNCTIONS
    hf = {k: v for k, v in cfg.to_hf_dict().items() if k not in ("model_type", "architectures")}
    want, scale = ROPE_INIT_FUNCTIONS["llama3"](transformers.LlamaConfig(**hf), "cpu")
    assert scale == 1.0
    assert torch.equal(inv, want.float())


def test_presets_have_no_scaling_unless_llama3():
    for name, cfg in PRESETS.items():
        scaled = name in ("llama-3.1-8b", "llama-3.2-1b", "llama-3.2-3b", "tiny-llama31")
        assert bool(cfg.rope_scaling) == scaled, name
        assert (rope_inv_freq(cfg) is None) != scaled, name
    for alias, name in (("meta-llama/Llama-3.1-8B", "llama-3.1-8b"), ("meta-llama/Llama-3.1-8B-Instruct", "llama-3.1-8b"),
                        ("llama3.1", "llama-3.1-8b"), ("meta-llama/Llama-3.2-1B-Instruct", "llama-3.2-1b"),
                        ("meta-llama/Llama-3.2-3B", "llama-3.2-3b"), ("llama3", "llama-3-8b")):
        assert resolve_config(alias).name == name, alias


@pytest.mark.parametrize("layout", ["rope_scaling", "rope_parameters"])
def test_published_configs_parse(layout):
    for d, preset, eos in ((LLAMA31_8B_INSTRUCT, "llama-3.1-8b", (128001, 128008, 128009)),
                           (LLAMA32_3B, "llama-3.2-3b", (128001,))):
        src = d if layout == "rope_scaling" else _as_rope_parameters(d)
        cfg = ModelConfig.from_hf_dict(json.loads(json.dumps(src)), name=preset)
        want = PRESETS[preset]
        assert dataclasses.replace(cfg, eos_token_ids=want.eos_token_ids) == want
        assert cfg.eos_token_id == 128001 and cfg.eos_token_ids == eos and cfg.eos_ids == eos
        assert torch.equal(rope_inv_freq(cfg), rope_inv_freq(want))
        # written back, read again: the same config, and transformers reads the same frequencies
        back = ModelConfig.from_hf_dict(json.loads(json.dumps(cfg.to_hf_dict())), name=preset)
        assert back == cfg


def test_single_eos_and_plain_rope_unchanged():
    tiny = resolve_config("tiny-llama")
    cfg = ModelConfig.from_hf_dict(tiny.to_hf_dict(), name="tiny-llama")
    assert cfg.rope_scaling is None and cfg.eos_ids == (tiny.eos_token_id,) and tiny.eos_ids == (tiny.eos_token_id,)
    assert "rope_scaling" not in tiny.to_hf_dict() and tiny.to_hf_dict()["eos_token_id"] == tiny.eos_token_id
    default = ModelConfig.from_hf_dict({**tiny.to_hf_dict(), "rope_scaling": {"rope_type": "default"}})
    assert default.rope_scaling is None
    v5 = {**tiny.to_hf_dict(), "rope_theta": None, "rope_parameters": {"rope_type": "default", "rope_theta": 1234.0}}
    assert ModelConfig.from_hf_dict(v5).rope_theta == 1234.0


@pytest.mark.parametrize("drop", ["factor", "low_freq_factor", "high_freq_factor", "original_max_position_embeddings"])
def test_incomplete_llama3_raises_and_names_the_key(drop):
    base = resolve_config("tiny-llama31").to_hf_dict()
    rs = {k: v for k, v in base["rope_scaling"].items() if k != drop}
    with pytest.raises(ValueError, match=drop):
        ModelConfig.from_hf_dict({**base, "rope_scaling": rs})
    with pytest.raises(ValueError, match=drop):
        ModelConfig.from_hf_dict(_as_rope_parameters({**base, "rope_scaling": rs}))


@pytest.mark.parametrize("rs", [{"rope_type": "llama3", "factor": 8.0},
                                {"rope_type": "llama3", "factor": 8.0, "low_freq_factor": 4.0, "high_freq_factor": 1.0,
                                 "original_max_position_embeddings": 8192},
                                {"rope_type": "linear", "factor": 2.0}, {"type": "dynamic", "factor": 2.0},
                                {"rope_type": "yarn", "factor": 4.0, "original_max_position_embeddings": 32768},
                                {"rope_type": "longrope", "short_factor": [1.0], "long_factor": [1.0]},
                                {"rope_type": "something-new"}])
def test_other_rope_types_raise(rs):
    base = resolve_config("tiny-llama").to_hf_dict()
    with pytest.raises(ValueError):
        ModelConfig.from_hf_dict({**base, "rope_scaling": rs})
    with pytest.raises(ValueError):
        ModelConfig.from_hf_dict({**base, "rope_parameters": {**rs, "rope_theta": 10000.0}})
    with pytest.raises(ValueError):
        ModelConfig.from_hf_dict({**LLAMA31_8B_INSTRUCT, "attention_bias": True})


def test_oracle_matches_transformers_past_the_original_context(tmp_path):
    """tiny-llama31 (original context 64) at 300 tokens against LlamaForCausalLM read from the directory save_hf_dir
    wrote, whole and through the KV cache; the same oracle with plain RoPE does not match"""
    transformers = pytest.importorskip("transformers")
    cfg = resolve_config("tiny-llama31")
    t = init_random(cfg, range(cfg.n_layers), True, True, seed=2)
    save_hf_dir(str(tmp_path), cfg, t, dtype=torch.float32)
    assert resolve_config(str(tmp_path)).rope_scaling == cfg.rope_scaling
    hf = transformers.AutoModelForCausalLM.from_pretrained(str(tmp_path), dtype=torch.float32,
                                                          attn_implementation="eager").eval()
    g = torch.Generator().manual_seed(0)
    ids = torch.randint(0, cfg.vocab_size, (2, 300), generator=g)
    pos = torch.arange(300)[None].expand(2, -1)
    with torch.no_grad():
        ref = hf(input_ids=ids).logits
    ours = TorchPiece(cfg, range(cfg.n_layers), True, True, t).forward(ids, pos, None)
    assert torch.allclose(ours, ref, atol=2e-4, rtol=2e-3), (ours - ref).abs().max()
    piece = TorchPiece(cfg, range(cfg.n_layers), True, True, t)
    cache = piece.new_cache()
    parts = [piece.forward(ids[:, :200], pos[:, :200], cache)]
    parts += [piece.forward(ids[:, i:i + 1], pos[:, i:i + 1], cache) for i in range(200, 300)]
    assert torch.allclose(torch.cat(parts, 1), ref, atol=2e-4, rtol=2e-3)
    plain = TorchPiece(dataclasses.replace(cfg, rope_scaling=None), range(cfg.n_layers), True, True, t)
    assert not torch.allclose(plain.forward(ids, pos, None), ref, atol=2e-4, rtol=2e-3)


def _eos_dir(tmp_path, name, eos):
    cfg = resolve_config("tiny-llama31")
    d = tmp_path / name
    save_hf_dir(str(d), cfg, init_random(cfg, range(cfg.n_layers), True, True, seed=5), dtype=torch.float32)
    c = json.loads((d / "config.json").read_text())
    c["eos_token_id"] = eos
    (d / "config.json").write_text(json.dumps(c))
    return str(d)


def _run(eng, prompt, sp):
    req = eng.submit(prompt, sp)
    while not req.done.is_set():
        eng.step()
    return req


def test_engine_stops_at_every_listed_eos(tmp_path):
    prompt = [3, 17, 99, 4, 250, 8]
    free = Engine(_eos_dir(tmp_path, "llama31-free", []), device="cpu", max_batch=2, max_seq_len=128).generate(
        [prompt], SamplingParams(max_new_tokens=16, temperature=0.0))[0]
    assert len(free) == 16
    unused = [t for t in range(2, 512) if t not in free][:2]
    for pick in (2, 3):                    # stop on the second, then on the third id of the list
        stop = free[6]
        eos = [unused[0], stop, unused[1]] if pick == 2 else [unused[0], unused[1], stop]
        d = _eos_dir(tmp_path, f"llama31-eos{pick}", eos)
        eng = Engine(d, device="cpu", max_batch=2, max_seq_len=128)
        assert eng.cfg.eos_token_id == unused[0] and eng.cfg.eos_ids == tuple(eos)
        req = _run(eng, prompt, SamplingParams(max_new_tokens=16, temperature=0.0))
        assert req.out_ids == free[:free.index(stop) + 1] and req.finish_reason == "stop"
        req = _run(eng, prompt, SamplingParams(max_new_tokens=16, temperature=0.0, ignore_eos=True))
        assert req.out_ids == free and req.finish_reason == "length"


def test_hf_service_serves_a_llama31_directory(tmp_path):
    """``serve-hf --model <dir>`` on a Llama-3.1-shaped directory: the service loads it and answers, and with a
    three-id EOS list whose last id is the fourth generated token the answer ends at that token"""
    from bee2bee_b200.hf import generate_text, load_model_and_tokenizer, unload_model
    from bee2bee_b200.services import HFService

    free_dir = _eos_dir(tmp_path, "llama31-free", [])          # no EOS: runs to max_new_tokens
    lm, tok, dev = load_model_and_tokenizer(free_dir, "cpu", max_batch=2, max_seq_len=128)
    try:
        _, ids = generate_text(lm, tok, dev, "hello there", 12, temperature=0.0, return_ids=True)
    finally:
        unload_model(free_dir)
    assert len(ids) == 12
    stop = ids[3]
    other = [t for t in range(2, 512) if t not in ids][:2]
    d = _eos_dir(tmp_path, "llama31-eot", [other[0], other[1], stop])
    svc = HFService(d, 0.0, max_batch=2, max_seq_len=128, device="cpu")
    svc.load_sync()
    try:
        r = svc.execute({"prompt": "hello there", "max_new_tokens": 12, "temperature": 0})
    finally:
        unload_model(d)
    assert r["tokens"] == ids.index(stop) + 1 and isinstance(r["text"], str)


def test_nccl_comparator_refuses_scaled_rope():
    from baseline.nccl_pipeline import NcclPipeline
    with pytest.raises(ValueError, match="rope_scaling"):
        NcclPipeline("tiny-llama31", 0, 1, torch.device("cpu"), 1, 1, 64)
