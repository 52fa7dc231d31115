"""Presence and frequency penalties from the request surfaces down to ``SamplingParams`` (CPU): validation, the
reference sampler, the CPU backend's counts, /generate and /chat (local and relayed), the Ollama options, and the mesh
``gen_request`` message."""
import asyncio

import numpy as np
import pytest
import torch
from fastapi.testclient import TestClient

from bee2bee_b200 import api as api_mod
from bee2bee_b200 import protocol as P
from bee2bee_b200.engine.core import Engine, SamplingParams
from bee2bee_b200.engine.runner import SeqInit
from bee2bee_b200.models.torch_ref import COUNT_MAX, sample_reference
from bee2bee_b200.p2p_runtime import P2PNode
from bee2bee_b200.services import EmbeddedOllama, HFService, sampling_filters

PROMPTS = [[1, 5, 9, 33, 2, 7], [4, 4, 19]]
PF = ("presence_penalty", "frequency_penalty")


def _record_submits(engine):
    """wrap ``engine.submit`` so every SamplingParams it receives is kept"""
    seen = []
    orig = engine.submit

    def submit(ids, params=None, on_token=None):
        seen.append(params)
        return orig(ids, params, on_token)

    engine.submit = submit
    return seen


def _pf(sp):
    return sp.presence_penalty, sp.frequency_penalty


def test_submit_validates_penalties():
    eng = Engine("tiny-llama", device="cpu", max_batch=2, max_seq_len=64)
    for name in PF:
        for bad in (float("nan"), float("inf"), -float("inf"), 2.0001, -2.5, 3.0):
            with pytest.raises(ValueError):
                eng.submit([1, 2, 3], SamplingParams(max_new_tokens=2, **{name: bad}))
    assert _pf(SamplingParams()) == (0.0, 0.0)
    out = eng.generate([[1, 2, 3]], SamplingParams(max_new_tokens=3, presence_penalty=-2.0, frequency_penalty=2.0,
                                                   ignore_eos=True))
    assert len(out[0]) == 3


def _direct(raw, seen, counts, pen, pres, freq):
    """the penalised logits in float32, step by step as the kernel states them"""
    l = raw.astype(np.float32).copy()
    pl = np.where(l > 0, l / np.float32(pen), l * np.float32(pen)).astype(np.float32)
    l = np.where(seen, pl, l) if pen != 1.0 else l
    c = counts.astype(np.float32)
    step = (l - np.float32(freq) * c).astype(np.float32) - np.float32(pres)
    return np.where(counts > 0, step, l).astype(np.float32)


def test_sample_reference_applies_penalties_after_repetition_penalty():
    rng = np.random.default_rng(0)
    V = 600
    for i in range(12):
        raw = (rng.standard_normal(V) * 3).astype(np.float32)
        seen = rng.random(V) < 0.1
        counts = np.where(rng.random(V) < 0.2, rng.integers(1, 40, V), 0).astype(np.int32)
        counts[:3] = (COUNT_MAX, 1, 0)
        pen = (1.0, 1.3)[i % 2]
        pres, freq = ((0.5, 0.0), (0.0, 0.7), (1.5, 0.25), (-0.8, -0.1))[i % 4]
        want = _direct(raw, seen, counts, pen, pres, freq)
        # greedy: the argmax of the penalised row
        got = sample_reference(torch.from_numpy(raw)[None], torch.from_numpy(seen)[None], 0.0, 1.0, pen,
                               counts=torch.from_numpy(counts)[None], presence=pres, frequency=freq)
        assert int(got) == int(np.argmax(want)), i
        # sampled with top_k = 1 keeps the argmax of the penalised row too
        got = sample_reference(torch.from_numpy(raw)[None], torch.from_numpy(seen)[None], 0.9, 1.0, pen,
                               torch.Generator().manual_seed(i), top_k=1, counts=torch.from_numpy(counts)[None],
                               presence=pres, frequency=freq)
        assert int(got) == int(np.argmax(want)), i
    # a token that the penalty moves off the argmax, and one that a negative penalty moves onto it
    raw = np.zeros(V, np.float32)
    raw[10], raw[20] = 5.0, 4.0
    counts = np.zeros(V, np.int32)
    counts[10] = 3
    args = (torch.from_numpy(raw)[None], None, 0.0, 1.0, 1.0)
    assert int(sample_reference(*args)) == 10
    assert int(sample_reference(*args, counts=torch.from_numpy(counts)[None], frequency=0.5)) == 20
    assert int(sample_reference(*args, counts=torch.from_numpy(counts)[None], presence=1.01)) == 20
    assert int(sample_reference(*args, counts=torch.from_numpy(counts)[None], presence=0.99)) == 10
    counts[10], counts[20] = 0, 1
    assert int(sample_reference(*args, counts=torch.from_numpy(counts)[None], presence=-1.5)) == 20
    # off: zero penalties or no counts give the draws of a call without them
    lg = torch.from_numpy((rng.standard_normal((3, 500)) * 2).astype(np.float32))
    c = torch.from_numpy(rng.integers(0, 5, (3, 500)).astype(np.int32))
    a = sample_reference(lg, None, 0.8, 0.9, 1.0, torch.Generator().manual_seed(1))
    b = sample_reference(lg, None, 0.8, 0.9, 1.0, torch.Generator().manual_seed(1), counts=c)
    d = sample_reference(lg, None, 0.8, 0.9, 1.0, torch.Generator().manual_seed(1), presence=1.0, frequency=1.0)
    assert torch.equal(a, b) and torch.equal(a, d)


def test_cpu_sequence_sampler_counts_generated_tokens_only():
    """the CPU backend's per-sequence counts (held by each sequence's ``SequenceSampler``) are the histogram of the
    generated tokens; prompt tokens are not counted, so a penalty changes nothing for the first token"""
    eng = Engine("tiny-llama", device="cpu", max_batch=2, max_seq_len=64)
    runner = eng.runner
    prompt = [7, 7, 7, 3, 3, 9]
    kw = dict(prompt=prompt, pages=[], temperature=0.0, top_p=1.0, repetition_penalty=1.0)
    runner.prefill([SeqInit(slot=0, presence_penalty=2.0, frequency_penalty=2.0, **kw), SeqInit(slot=1, **kw)])
    runner.decode(9)
    pen, plain = runner.state[0]["hist"], runner.state[1]["hist"]
    hist = {}
    for t in pen:
        hist[t] = hist.get(t, 0) + 1
    counts = runner.state[0]["sampler"].counts[0]
    assert {int(t): int(counts[t]) for t in counts.nonzero()} == hist
    assert sum(hist.values()) == len(pen) == 10
    assert plain[0] == pen[0]                       # counts start empty: the prompt is not penalised
    assert plain != pen                             # and the penalties do act on generated tokens
    assert max(hist.values()) < max(plain.count(t) for t in set(plain))


def test_sampling_filters_carries_penalties_only_when_set():
    assert sampling_filters({}) == {}
    assert sampling_filters({"presence_penalty": None, "frequency_penalty": None}) == {}
    assert sampling_filters({"presence_penalty": 1, "frequency_penalty": "-0.5"}) == {"presence_penalty": 1.0,
                                                                                      "frequency_penalty": -0.5}
    assert sampling_filters({"frequency_penalty": 0.0}) == {"frequency_penalty": 0.0}


def test_ollama_options_reach_sampling_params():
    ol = EmbeddedOllama("tiny-llama", max_batch=2, max_seq_len=64, device="cpu")
    seen = _record_submits(ol._ensure().engine)
    opts = {"num_predict": 2, "presence_penalty": 0.6, "frequency_penalty": -0.4}
    list(ol.generate({"prompt": "hi", "stream": False, "options": opts}))
    list(ol.generate({"prompt": "hi", "stream": False, "options": {"num_predict": 2}}))
    list(ol.generate({"prompt": "hi", "stream": False, "options": {"num_predict": 2, "frequency_penalty": 1.0,
                                                                    "top_k": -1}}))
    assert _pf(seen[0]) == (0.6, -0.4)                # negative values favour repetition; they are not turned off
    assert _pf(seen[1]) == (0.0, 0.0)
    assert (seen[1].temperature, seen[1].top_p, seen[1].repetition_penalty) == (0.8, 0.9, 1.1)
    assert _pf(seen[2]) == (0.0, 1.0) and seen[2].top_k == 0


def test_gen_request_without_penalties_is_unchanged():
    base = {"type": "gen_request", "rid": "r", "prompt": "p", "model": "m", "svc": "hf", "max_new_tokens": 5,
            "max_tokens": 5, "temperature": 0.3, "stream": True}
    m = P.gen_request("r", "p", model="m", max_new_tokens=5, temperature=0.3, stream=True)
    assert m == base and list(m) == list(base)
    m = P.gen_request("r", "p", model="m", max_new_tokens=5, temperature=0.3, stream=True, presence_penalty=0.5,
                      frequency_penalty=-1)
    assert m == {**base, "presence_penalty": 0.5, "frequency_penalty": -1.0}
    assert P.gen_request("r", "p", frequency_penalty=0.2) == {**P.gen_request("r", "p"), "frequency_penalty": 0.2}


@pytest.fixture()
def client(monkeypatch):
    monkeypatch.setenv("BEE2BEE_TRANSPORT", "inproc")
    monkeypatch.delenv("BEE2BEE_API_KEY", raising=False)
    api_mod.node = None
    with TestClient(api_mod.app) as c:
        yield c
    api_mod.node = None


def test_generate_and_chat_penalties_reach_sampling_params_local(client):
    svc = HFService("tiny-llama", 0.0, max_batch=2, max_seq_len=128, device="cpu")
    svc.load_sync()
    api_mod.node.local_services["hf"] = svc
    seen = _record_submits(svc.model.engine)
    try:
        body = {"prompt": "user: hi", "max_new_tokens": 2, "temperature": 0.5}
        r = client.post("/generate", json={**body, "presence_penalty": 0.5, "frequency_penalty": 0.25})
        assert r.json()["status"] == "ok"
        assert client.post("/chat", json={**body, "frequency_penalty": -1.0}).json()["status"] == "ok"
        assert client.post("/chat", json=body).json()["status"] == "ok"
        with client.stream("POST", "/generate", json={**body, "stream": True, "presence_penalty": 1.5}) as resp:
            list(resp.iter_lines())
        assert client.post("/generate", json={**body, "presence_penalty": 2.5}).json()["status"] == "error"
    finally:
        svc.model.engine.stop()
    assert [_pf(s) for s in seen[:4]] == [(0.5, 0.25), (0.0, -1.0), (0.0, 0.0), (1.5, 0.0)]
    assert seen[0].top_p == 1.0 and seen[3].top_p == 0.95      # the paths' own defaults are unchanged


def test_generate_and_chat_penalties_reach_remote_provider(client, monkeypatch):
    calls = []

    async def fake_request_generation(pid, prompt, max_new_tokens=32, model_name=None, **kw):
        calls.append(kw)
        return {"text": "ok"}

    monkeypatch.setattr(api_mod.node, "request_generation", fake_request_generation)
    body = {"prompt": "x", "provider_id": "peer-elsewhere", "max_new_tokens": 3}
    assert client.post("/generate", json={**body, "presence_penalty": 0.3}).json()["status"] == "ok"
    assert client.post("/chat", json={**body, "frequency_penalty": 0.4, "top_k": 2}).json()["status"] == "ok"
    assert client.post("/generate", json=body).json()["status"] == "ok"
    assert calls[0] == {"temperature": 0.7, "presence_penalty": 0.3}
    assert calls[1] == {"temperature": 0.7, "top_k": 2, "frequency_penalty": 0.4}
    assert calls[2] == {"temperature": 0.7}


def test_mesh_requests_and_relay_carry_penalties():
    """requester -> provider, requester -> relay -> provider, and a streamed request: the provider's engine receives
    the penalties; a request without them reaches it with both off"""
    async def go():
        nodes = [P2PNode(host="127.0.0.1", port=0, transport="inproc", name=f"pf{i}-{id(object())}",
                         health_interval=0.2, pong_timeout=1.0) for i in range(3)]
        for nd in nodes:
            await nd.start()
        a, b, c = nodes
        svc = HFService("tiny-llama", 0.0, max_batch=2, max_seq_len=128, device="cpu")
        svc.load_sync()
        seen = _record_submits(svc.model.engine)
        try:
            await b.add_service(svc)
            await a.connect_bootstrap(b.addr)
            await c.connect_bootstrap(a.addr)
            t0 = asyncio.get_running_loop().time()
            while not (b.peer_id in a.providers and len(c.peers) == 2):
                assert asyncio.get_running_loop().time() - t0 < 10
                await asyncio.sleep(0.01)
            await a.request_generation(b.peer_id, "hello", 2, "tiny-llama", presence_penalty=0.7,
                                       frequency_penalty=0.1, timeout=60)
            await a.request_generation(b.peer_id, "hello", 2, "tiny-llama", timeout=60)
            await a.request_generation(b.peer_id, "user: hi", 2, "tiny-llama", frequency_penalty=-0.3,
                                       on_chunk=lambda s: None, timeout=60)
            # relay: c asks a, which does not serve the model and forwards to b
            await c._drop_peer(b.peer_id)
            c.providers.pop(b.peer_id, None)
            fut = asyncio.get_running_loop().create_future()
            c._pending_requests["r1"] = fut
            await c._send(c._conn_of(a.peer_id), P.gen_request("r1", "relay", model="tiny-llama", max_new_tokens=2,
                                                                presence_penalty=1.25))
            out = await asyncio.wait_for(fut, 60)
            assert not out.get("error"), out
        finally:
            svc.model.engine.stop()
            for n in nodes:
                await n.stop()
        return seen

    seen = asyncio.run(go())
    assert [_pf(s) for s in seen] == [(0.7, 0.1), (0.0, 0.0), (0.0, -0.3), (1.25, 0.0)]
