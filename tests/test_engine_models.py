"""Engine / model layer on CPU: configs, piece splitting, weights round trip, the torch oracle
against Hugging Face's own modelling code, tokenizer, scheduler behaviour."""
import math
import os

import pytest
import torch

from bee2bee_b200.engine.core import Engine, SamplingParams
from bee2bee_b200.engine.kv import OutOfPages, PageAllocator
from bee2bee_b200.engine.tokenizer import ByteTokenizer, cut_at_stop_words, parse_transcript
from bee2bee_b200.models.config import PRESETS, ModelConfig, resolve_config, split_layers
from bee2bee_b200.models.torch_ref import TorchPiece, sample_reference, top_p_keep_mask
from bee2bee_b200.models.weights import init_random, load_hf_dir, save_hf_dir


def test_presets_match_public_architectures():
    l = resolve_config("meta-llama/Meta-Llama-3-8B")
    assert (l.n_layers, l.hidden_size, l.n_heads, l.n_kv_heads, l.head_dim, l.ffn_size, l.vocab_size) == \
        (32, 4096, 32, 8, 128, 14336, 128256)
    assert 7.9e9 < l.param_count() < 8.1e9
    g = resolve_config("gemma2:2b")
    assert (g.n_layers, g.hidden_size, g.head_dim, g.n_heads, g.n_kv_heads) == (26, 2304, 256, 8, 4)
    assert g.layer_window(0) == 4096 and g.layer_window(1) == 0 and g.attn_softcap == 50.0 and g.post_norms
    z = resolve_config("HuggingFaceH4/zephyr-7b-beta")
    assert z.family == "mistral" and z.sliding_window == 4096 and z.vocab_size == 32000
    d = resolve_config("distilgpt2")
    assert (d.n_layers, d.hidden_size, d.n_heads, d.head_dim, d.vocab_size) == (6, 768, 12, 64, 50257) and d.bias
    with pytest.raises(KeyError):
        resolve_config("no-such-model")


def test_split_layers_uneven():
    assert [len(r) for r in split_layers(26, 4)] == [7, 7, 6, 6]
    assert [len(r) for r in split_layers(32, 8)] == [4] * 8
    assert [list(r) for r in split_layers(6, 2)] == [[0, 1, 2], [3, 4, 5]]
    assert len(split_layers(2, 8)) == 2


def test_random_init_is_piece_invariant():
    cfg = resolve_config("tiny-llama")
    whole = init_random(cfg, range(4), True, True, seed=3)
    part = init_random(cfg, range(2, 4), False, True, seed=3)
    for k, v in part.items():
        assert torch.equal(v, whole[k]), k
    assert "embed" not in part and "lm_head" in part
    assert not torch.equal(init_random(cfg, range(1), True, False, seed=4)["embed"], whole["embed"])


@pytest.mark.parametrize("name", ["tiny-llama", "tiny-gpt2", "tiny-gemma2", "tiny-mistral"])
def test_hf_directory_roundtrip(name, tmp_path):
    cfg = resolve_config(name)
    t = init_random(cfg, range(cfg.n_layers), True, True, seed=1)
    save_hf_dir(str(tmp_path), cfg, t, dtype=torch.float32)
    cfg2 = resolve_config(str(tmp_path))
    assert (cfg2.family, cfg2.n_layers, cfg2.hidden_size, cfg2.head_dim) == (cfg.family, cfg.n_layers, cfg.hidden_size, cfg.head_dim)
    back = load_hf_dir(str(tmp_path), cfg2, range(1, 3), False, False)
    assert back is not None and all(k.startswith(("l1.", "l2.")) for k in back)
    for k, v in back.items():
        assert torch.allclose(v, t[k]), k


@pytest.mark.parametrize("name", ["tiny-llama", "tiny-gpt2", "tiny-gemma2", "tiny-mistral"])
def test_oracle_matches_transformers(name, tmp_path):
    """Our plain-torch model == HF's modelling code on the same random weights (validates the
    oracle every CUDA kernel is tested against)."""
    transformers = pytest.importorskip("transformers")
    cfg = resolve_config(name)
    t = init_random(cfg, range(cfg.n_layers), True, True, seed=2)
    save_hf_dir(str(tmp_path), cfg, t, dtype=torch.float32)
    hf = transformers.AutoModelForCausalLM.from_pretrained(str(tmp_path), dtype=torch.float32, attn_implementation="eager").eval()
    ids = torch.tensor([[5, 9, 2, 77, 130, 8, 41, 3, 3, 250, 17, 99]])
    pos = torch.arange(ids.shape[1])[None]
    ours = TorchPiece(cfg, range(cfg.n_layers), True, True, t).forward(ids, pos, None)
    with torch.no_grad():
        ref = hf(input_ids=ids).logits
    assert torch.allclose(ours, ref, atol=2e-4, rtol=2e-3), (ours - ref).abs().max()
    # incremental decoding through our KV cache reproduces the full-sequence logits
    piece = TorchPiece(cfg, range(cfg.n_layers), True, True, t)
    cache = piece.new_cache()
    a = piece.forward(ids[:, :7], pos[:, :7], cache)
    b = piece.forward(ids[:, 7:], pos[:, 7:], cache)
    assert torch.allclose(torch.cat([a, b], 1), ours, atol=2e-4, rtol=2e-3)


def test_sliding_window_changes_long_range_attention():
    cfg = resolve_config("tiny-mistral")           # window 96
    t = init_random(cfg, range(cfg.n_layers), True, True)
    piece = TorchPiece(cfg, range(cfg.n_layers), True, True, t)
    ids = torch.randint(0, cfg.vocab_size, (1, 150))
    ids2 = ids.clone()
    ids2[0, 0] = (ids2[0, 0] + 1) % cfg.vocab_size
    pos = torch.arange(150)[None]
    a, b = piece.forward(ids, pos, None), piece.forward(ids2, pos, None)
    assert not torch.allclose(a[0, 50], b[0, 50])          # token 0 is inside the window of position 50
    # position 149 can still be influenced through stacked layers (4 x 96 > 149) -- but a single layer cannot:
    one = TorchPiece(cfg, range(1), True, False, t)
    ha, hb = one.forward(ids, pos, None), one.forward(ids2, pos, None)
    assert torch.allclose(ha[0, 149], hb[0, 149]) and not torch.allclose(ha[0, 90], hb[0, 90])


def test_sampler_reference_semantics():
    torch.manual_seed(0)
    logits = torch.randn(4, 300) * 3
    seen = torch.zeros(4, 300, dtype=torch.bool)
    assert torch.equal(sample_reference(logits, seen, 0.0, 0.95, 1.15), logits.argmax(-1))    # greedy iff T <= 0
    top = logits.argmax(-1)
    seen[torch.arange(4), top] = True
    pen = sample_reference(logits, seen, 0.0, 1.0, 100.0)
    assert (pen != top).all()                                   # heavily penalised arg-max loses
    keep = top_p_keep_mask(logits, 0.7, 0.95)
    g = torch.Generator().manual_seed(1)
    for _ in range(50):
        tok = sample_reference(logits, None, 0.7, 0.95, 1.0, g)
        assert keep[torch.arange(4), tok].all()
    p = (logits / 0.7).softmax(-1)
    assert ((p * keep).sum(-1) >= 0.95 - 1e-6).all() and (keep.sum(-1) < 300).all()


def test_byte_tokenizer_and_transcript_helpers():
    tok = ByteTokenizer(50257, eos_id=50256, bos_id=50256)
    ids = tok.encode("héllo wörld")
    assert ids[0] == 50256 and tok.decode(ids) == "héllo wörld"
    assert tok.decode([70000, 4 + 65]) != ""           # out-of-range ids still render something printable
    small = ByteTokenizer(384)
    assert all(0 <= i < 384 for i in small.encode("any text at all"))
    msgs = parse_transcript("system: be brief\nuser: hi\nthere\nassistant: hello\nuser: bye\nassistant:")
    assert [m["role"] for m in msgs] == ["system", "user", "assistant", "user"]
    assert msgs[1]["content"] == "hi\nthere"
    assert parse_transcript("just text") == [{"role": "user", "content": "just text"}]
    assert cut_at_stop_words("fine answer\nuser: next") == ("fine answer\n", True)
    assert cut_at_stop_words("no stop here") == ("no stop here", False)
    assert "<|assistant|>" in tok.apply_chat_template(msgs)


def test_page_allocator():
    a = PageAllocator(10)
    assert a.free_pages == 9 and a.pages_for(64) == 1 and a.pages_for(65) == 2
    p = a.allocate(1, 130)
    assert len(p) == 3 and 0 not in p
    assert a.can_allocate(6 * 64) and not a.can_allocate(7 * 64)
    with pytest.raises(OutOfPages):
        a.allocate(2, 7 * 64)
    a.release(1)
    assert a.free_pages == 9 and a.utilization() == 0.0


def test_engine_continuous_batching_and_limits():
    eng = Engine("tiny-llama", device="cpu", max_batch=2, max_seq_len=64)
    sp = SamplingParams(max_new_tokens=5, temperature=0.0, ignore_eos=True)
    prompts = [[1, 2, 3], [4, 5], [6], [7, 8, 9, 10]]            # 4 requests through 2 slots
    outs = eng.generate(prompts, sp)
    assert [len(o) for o in outs] == [5, 5, 5, 5]
    solo = Engine("tiny-llama", device="cpu", max_batch=1, max_seq_len=64)
    assert solo.generate([prompts[2]], sp)[0] == outs[2]          # batching does not change results
    # context budget: prompt is truncated from the left, generation clipped
    long = eng.generate([list(range(100))], SamplingParams(max_new_tokens=50, temperature=0.0, ignore_eos=True))[0]
    assert 1 <= len(long) <= 50
    m = eng.metrics()
    assert m["requests"] == 5 and m["tokens_generated"] == 20 + len(long) and m["running"] == 0
    assert eng.alloc.free_pages == eng.alloc.num_pages - 1       # every page returned


def test_engine_eos_stop_and_streaming_thread():
    eng = Engine("tiny-gpt2", device="cpu", max_batch=2, max_seq_len=64)
    first = eng.generate([[3, 4, 5]], SamplingParams(max_new_tokens=6, temperature=0.0, ignore_eos=True))[0]
    stop = first[2]
    r = eng.generate([[3, 4, 5]], SamplingParams(max_new_tokens=6, temperature=0.0, ignore_eos=True,
                                                 stop_token_ids=(stop,)))[0]
    assert r == first[:first.index(stop) + 1]
    got = []
    eng.start()
    req = eng.submit([3, 4, 5], SamplingParams(max_new_tokens=6, temperature=0.0, ignore_eos=True), on_token=got.append)
    req.wait(timeout=30)
    eng.stop()
    assert got == first and req.finish_reason == "length" and req.ttft_ms > 0


def test_engine_cancel_frees_slot_and_pages():
    """ADVICE r1: an abandoned request (stop word / disconnect / timeout) must not decode to max_new_tokens"""
    eng = Engine("tiny-llama", device="cpu", max_batch=1, max_seq_len=256, decode_burst=2)
    sp = SamplingParams(max_new_tokens=200, temperature=0.0, ignore_eos=True)
    a = eng.submit([1, 2, 3], sp)
    b = eng.submit([4, 5], SamplingParams(max_new_tokens=3, temperature=0.0, ignore_eos=True))   # waits for the only slot
    eng.step()
    assert len(a.out_ids) >= 1 and not a.done.is_set() and not b.done.is_set()
    eng.cancel(a)
    while not b.done.is_set():
        eng.step()
    assert a.done.is_set() and a.finish_reason == "cancelled" and len(a.out_ids) < 20
    assert len(b.out_ids) == 3
    assert eng.alloc.free_pages == eng.alloc.num_pages - 1 and len(eng._free_slots) == 1
    # cancelling a queued request removes it from the queue
    c = eng.submit([7], sp)
    d = eng.submit([8], sp)
    eng.step()
    eng.cancel(d)
    eng.cancel(c)
    eng.step()
    assert c.done.is_set() and d.done.is_set() and not eng._running and not eng._pending
    # the streaming helper cancels when its consumer walks away (generator closed)
    from bee2bee_b200 import hf
    lm, tok, _ = hf.load_model_and_tokenizer("tiny-llama", device="cpu")
    gen = hf.generate_text_stream(lm, tok, "cpu", "user: hi", max_new_tokens=400, temperature=0.0)
    next(gen)
    gen.close()
    import time
    t0 = time.time()
    while lm.engine._running and time.time() - t0 < 20:
        time.sleep(0.05)
    assert not lm.engine._running, "zombie request kept its slot"


def test_engine_prefill_failure_does_not_leak_requests():
    """ADVICE r1: admitted requests were lost (waiters hung, slot + pages leaked) when runner.prefill raised"""
    eng = Engine("tiny-llama", device="cpu", max_batch=2, max_seq_len=64)
    boom = {"n": 1}
    real = eng.runner.prefill

    def flaky(seqs):
        if boom["n"]:
            boom["n"] -= 1
            raise RuntimeError("injected prefill fault")
        return real(seqs)

    eng.runner.prefill = flaky
    r = eng.submit([1, 2, 3], SamplingParams(max_new_tokens=4, temperature=0.0, ignore_eos=True))
    with pytest.raises(RuntimeError):
        eng.step()
    assert r.done.is_set() and "prefill failed" in (r.error or "")
    assert eng.alloc.free_pages == eng.alloc.num_pages - 1 and len(eng._free_slots) == 2 and not eng._running
    assert len(eng.generate([[1, 2, 3]], SamplingParams(max_new_tokens=4, temperature=0.0, ignore_eos=True))[0]) == 4


def test_seeded_sampling_is_reproducible():
    sp = SamplingParams(max_new_tokens=8, temperature=0.9, seed=11, ignore_eos=True)
    a = Engine("tiny-llama", device="cpu", max_batch=2, max_seq_len=64).generate([[1, 2, 3]], sp)
    b = Engine("tiny-llama", device="cpu", max_batch=2, max_seq_len=64).generate([[1, 2, 3]], sp)
    c = Engine("tiny-llama", device="cpu", max_batch=2, max_seq_len=64).generate(
        [[1, 2, 3]], SamplingParams(max_new_tokens=8, temperature=0.9, seed=12, ignore_eos=True))
    assert a == b and a != c


# ------------------------------------------------------------------ piece planning / quantisation helpers (CPU)
def test_piece_units_cover_the_model_and_balance_the_wavefront():
    from bee2bee_b200.models.config import balanced_split, piece_units, supports_half_layer_pieces

    cfg = resolve_config("llama-3-8b")
    assert supports_half_layer_pieces(cfg)
    for n in (1, 2, 4, 8):
        units = piece_units(cfg, n)
        assert len(units) == n and units[0][0] == 0 and units[-1][1] == 3 * cfg.n_layers
        assert all(a[1] == b[0] for a, b in zip(units, units[1:])) and all(u1 > u0 for u0, u1 in units)
    # the last piece also streams the 1 GB lm_head: it gets the fewest units, nobody gets more than the mean + one layer
    u8 = piece_units(cfg, 8)
    sizes = [b - a for a, b in u8]
    assert sizes[-1] == min(sizes) and max(sizes) <= 13 and any(b % 3 for a, b in u8)   # cuts inside layers are used
    assert any(b % 3 == 2 for a, b in u8[:-1])           # ... including one between a gate/up and a down GEMM
    # whole-layer fallback for graphs whose boundary GEMMs are not the fused kinds (post-norms / LayerNorm)
    for name in ("gemma-2-2b", "distilgpt2"):
        c = resolve_config(name)
        assert not supports_half_layer_pieces(c)
        assert piece_units(c, 2) == [(3 * r.start, 3 * r.stop) for r in balanced_split(c, 2)]
    # explicit bounds (tests / experiments)
    tiny = resolve_config("tiny-llama")
    assert piece_units(tiny, 2, [0, 5, 12]) == [(0, 5), (5, 12)]
    with pytest.raises(AssertionError):
        piece_units(tiny, 2, [0, 13])


def test_mx_block_scaled_quantisation_roundtrip_cpu():
    """OCP-MX e4m3: one power-of-two scale per 32 K elements; the GEMM's scale-factor chunk layout is a pure permutation."""
    from bee2bee_b200 import ops

    torch.manual_seed(0)
    w = (torch.randn(256, 512) * 0.05 * torch.exp2(torch.randint(-5, 5, (256, 16)).float()).repeat_interleave(32, 1)).bfloat16()
    q, chunks = ops.quantize_weight_mxfp8(w)
    assert q.dtype == torch.float8_e4m3fn and chunks.dtype == torch.uint8 and chunks.numel() == (256 // 128) * (512 // 128) * 512
    sf = ops.mx_unchunk(chunks, 256, 512, 128)
    assert torch.equal(ops.mx_chunk_layout(sf), chunks)
    # byte (r % 32) * 16 + (r / 32) * 4 + k-block inside the 512-byte chunk of (row tile, 128-K chunk)
    r, kb = 200, 13
    off = ((r // 128) * 4 + kb // 4) * 512 + (r % 32) * 16 + ((r % 128) // 32) * 4 + kb % 4
    assert chunks[off] == sf[r, kb]
    deq = ops.mx_dequant(q, sf)
    blocks = w.float().view(256, 16, 32)
    amax = blocks.abs().amax(-1, keepdim=True)
    err = (deq.view(256, 16, 32) - blocks).abs()
    assert (err <= 0.0625 * blocks.abs() + 1e-3 * amax).all()
    # scales are the smallest powers of two that keep |q| <= 448
    scale = torch.exp2(sf.float() - 127)
    assert (amax.squeeze(-1) / scale <= 448.0 + 1e-3).all() and (amax.squeeze(-1) / (scale / 2) > 448.0 - 1e-3)[amax.squeeze(-1) > 0].all()


def test_split_k_heuristic_matches_the_measured_optimum():
    from unittest import mock

    from bee2bee_b200 import ops

    fake = mock.Mock(gemm_max_splitk=lambda bn, epi, stages=0: 8)
    shapes = dict(qkv=(6144, 4096), o=(4096, 4096), gu=(28672, 4096), down=(4096, 14336), head=(128256, 4096))
    with mock.patch.object(ops, "native", lambda: fake):
        pick = lambda bn, m: {k: ops.pick_splitk(n, m, kk, bn, 0) for k, (n, kk) in shapes.items()}
        assert pick(32, 32) == dict(qkv=4, o=4, gu=1, down=8, head=1)      # up to ~2 CTAs per SM
        assert pick(16, 1) == dict(qkv=4, o=4, gu=1, down=4, head=1)       # >= 4 token columns per CTA of the cluster
        assert all(v == 1 for v in pick(256, 4096).values())               # prefill: tiles already fill the machine
    # prefill chunks: (token tile, ring depth, split-K) per GEMM of a Llama-3-8B layer: under-filled GEMMs are split
    # along K until the machine is full instead of running two waves
    tile = lambda m: {k: ops.pick_prefill_tile(n, m, kk) for k, (n, kk) in shapes.items() if k != "head"}
    assert tile(512) == dict(qkv=(128, 3, 1), o=(128, 3, 2), gu=(256, 2, 1), down=(256, 0, 2))
    assert tile(256) == dict(qkv=(128, 3, 2), o=(128, 3, 2), gu=(128, 3, 1), down=(256, 0, 4))
    assert tile(1024) == dict(qkv=(256, 2, 1), o=(128, 3, 1), gu=(256, 2, 1), down=(256, 0, 1))
    assert all(v == (256, 2, 1) for v in tile(4096).values())
    assert ops.pick_prefill_tile(256, 512, 256) == (128, 3, 1)             # tiny models: too few k-blocks to split


def test_attention_kernel_choice():
    """the extension's one attention-kernel decision (host code, no launch): decode and prefill chunks of >= tc_min_q
    queries run on the tensor-core kernel when it supports the GQA layout; the fused e4m3 output needs that kernel
    without split-KV"""
    from bee2bee_b200 import ops

    uses = lambda max_q, use_tc=-1, g=4, d=128: ops.native().attention_uses_tc(max_q, 2 * g, 2, d, use_tc)  # noqa: E731
    old = ops.get_attn_tc_min_q()
    try:
        ops.set_attn_tc_min_q(16)
        assert [uses(q) for q in (0, 1, 2, 15, 16, 500)] == [False, True, False, False, True, True]
        assert all(uses(q, 1) for q in (0, 1, 2, 15)) and not any(uses(q, 0) for q in (1, 16))
        assert not any(uses(q, u, g=g) for q in (1, 16) for u in (-1, 1) for g in (3, 12, 32))
        assert not any(uses(q, u, d=96) for q in (1, 16) for u in (-1, 1))
        assert ops.attention_fuses_quant(1, 8, 2, 128, 1) and not ops.attention_fuses_quant(1, 8, 2, 128, 4)
        assert ops.attention_fuses_quant(16, 8, 2, 128, 4) and not ops.attention_fuses_quant(15, 8, 2, 128, 1)
        assert not ops.attention_fuses_quant(1, 24, 2, 128, 1)
        ops.set_attn_tc_min_q(0)
        assert not any(uses(q, u) for q in (1, 16) for u in (-1, 1))
        assert not ops.attention_fuses_quant(1, 8, 2, 128, 1)
    finally:
        ops.set_attn_tc_min_q(old)


def test_weights_policy_random_init_is_opt_in(monkeypatch, tmp_path):
    """ADVICE r1: `serve-hf --model llama-3-8b` must not silently serve noise"""
    from bee2bee_b200.models.weights import WEIGHT_SOURCE, WeightsUnavailable, load_or_init
    from bee2bee_b200.services import HFService, ServiceError

    cfg = resolve_config("distilgpt2")
    monkeypatch.setenv("B2B_ALLOW_RANDOM_WEIGHTS", "0")
    with pytest.raises(WeightsUnavailable):
        load_or_init("distilgpt2", cfg, range(1), True, False)
    svc = HFService("distilgpt2", device="cpu")
    with pytest.raises(ServiceError):
        svc.load_sync()
    tiny = resolve_config("tiny-llama")
    assert "l0.wq" in load_or_init("tiny-llama", tiny, range(1), True, False)        # test presets stay usable
    monkeypatch.setenv("B2B_ALLOW_RANDOM_WEIGHTS", "1")
    assert "l0.wq" in load_or_init("distilgpt2", cfg, range(1), True, False)
    assert WEIGHT_SOURCE["distilgpt2"] == "random-init"
    # unsupported checkpoint flavours are rejected, not mis-loaded
    from bee2bee_b200.models.config import ModelConfig
    base = tiny.to_hf_dict()
    with pytest.raises(ValueError):
        ModelConfig.from_hf_dict({**base, "attention_bias": True})
    with pytest.raises(ValueError):
        ModelConfig.from_hf_dict({**base, "rope_scaling": {"rope_type": "llama3", "factor": 8.0}})


def test_engine_marks_itself_broken_when_the_mesh_stalls():
    """SURVEY 5.3: a peer piece that stops answering must fail the in-flight requests and take the provider out of
    service (the reference drops the peer, p2p_runtime.py:396-410) -- not hang or kill the node."""
    from bee2bee_b200.engine.runner import MeshStalled

    eng = Engine("tiny-llama", device="cpu", max_batch=2, max_seq_len=64)
    real = eng.runner.decode
    eng.runner.decode = lambda n: (_ for _ in ()).throw(MeshStalled("rank 0: a peer piece did not publish"))
    eng.start()
    r = eng.submit([1, 2, 3], SamplingParams(max_new_tokens=8, temperature=0.0, ignore_eos=True))
    with pytest.raises(RuntimeError):
        r.wait(timeout=30)
    assert "engine error" in r.error and eng.broken and not eng.metrics()["healthy"]
    late = eng.submit([4, 5], SamplingParams(max_new_tokens=2))
    assert late.done.is_set() and "mesh unavailable" in late.error           # refused at once, nothing queues
    assert not eng._running and eng.alloc.free_pages == eng.alloc.num_pages - 1
    eng.stop()
    eng.runner.decode = real


def test_prefix_cache_allocator_shares_pins_and_evicts():
    """content-addressed prompt pages: share (ref-counted), keep after release (LRU), evict under pressure"""
    from bee2bee_b200.engine.kv import OutOfPages, PageAllocator

    a = PageAllocator(10)                                   # 9 usable pages
    p1 = list(range(200))
    pages1 = a.allocate(1, 260, p1)
    assert len(pages1) == 5 and a.cached_tokens(1) == 0
    a.commit(1, p1)                                         # 3 full prompt pages become shareable
    pages2 = a.allocate(2, 260, p1[:150] + [9, 9, 9])       # shares the first 2 pages (128 tokens), 3 fresh ones
    assert pages2[:2] == pages1[:2] and a.cached_tokens(2) == 128 and a.free_pages == 1
    assert not a.can_allocate(3 * 64)
    a.release(1)                                            # shared pages stay pinned by owner 2; page 3 stays cached
    assert a.free_pages == 4 and a.cache_stats()["evictable_pages"] == 1
    a.release(2)
    assert a.free_pages == 9
    pages3 = a.allocate(3, 200, p1)                         # whole prompt minus its last token is resident: 3 pages
    assert pages3[:3] == pages1[:3] and a.cached_tokens(3) == 192
    a.release(3)
    big = a.allocate(4, 9 * 64)                             # pressure: every cached page is evicted
    assert len(big) == 9 and a.cache_stats()["cached_pages"] == 0
    with pytest.raises(OutOfPages):
        a.allocate(5, 64)
    # a prompt that fits exactly into full pages still prefills its last token
    b = PageAllocator(10)
    q = list(range(128))
    b.allocate(1, 192, q); b.commit(1, q); b.release(1)
    b.allocate(2, 192, q)
    assert b.cached_tokens(2) == 64
    # invalidate: pages of a failed prefill lose their keys
    c = PageAllocator(10)
    c.allocate(1, 192, q); c.commit(1, q); c.invalidate(1); c.release(1)
    c.allocate(2, 192, q)
    assert c.cached_tokens(2) == 0
    # the CPU backend (dense per-slot KV) never shares
    d = PageAllocator(10, prefix_cache=False)
    d.allocate(1, 192, q); d.commit(1, q); d.release(1); d.allocate(2, 192, q)
    assert d.cached_tokens(2) == 0


def test_request_deadline_frees_slot_and_pages():
    """VERDICT r1 #9: 'timeout -> slot + pages freed at the next burst boundary'.  A request past its ``timeout_s`` is
    retired with finish_reason "timeout" whether it is still queued or already decoding; the others are unaffected."""
    import time
    eng = Engine("tiny-llama", device="cpu", max_batch=1, max_seq_len=256, decode_burst=2)
    slow = eng.submit([1, 2, 3], SamplingParams(max_new_tokens=200, temperature=0.0, ignore_eos=True, timeout_s=0.05))
    queued = eng.submit([4, 5], SamplingParams(max_new_tokens=200, temperature=0.0, ignore_eos=True, timeout_s=0.05))
    ok = eng.submit([6, 7], SamplingParams(max_new_tokens=3, temperature=0.0, ignore_eos=True))
    eng.step()
    assert not slow.done.is_set() and len(slow.out_ids) >= 1
    time.sleep(0.08)
    while not ok.done.is_set():
        eng.step()
    assert slow.finish_reason == "timeout" and queued.finish_reason == "timeout" and not queued.out_ids
    assert len(slow.out_ids) < 200 and len(ok.out_ids) == 3 and ok.finish_reason == "length"
    assert eng.alloc.free_pages == eng.alloc.num_pages - 1 and len(eng._free_slots) == 1
    assert eng.metrics()["timeouts"] == 2 and eng.metrics()["cancelled"] >= 1
    # engine-wide default deadline
    eng.default_timeout_s = 0.01
    r = eng.submit([1], SamplingParams(max_new_tokens=500, temperature=0.0, ignore_eos=True))
    eng.step()
    time.sleep(0.03)
    eng.step()
    assert r.done.is_set() and r.finish_reason == "timeout"
