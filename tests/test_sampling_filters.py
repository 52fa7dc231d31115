"""Top-k and min-p from the request surfaces down to ``SamplingParams`` (CPU): validation, the CPU backend, /generate
(local and relayed), the Ollama options, and the mesh ``gen_request`` message."""
import asyncio

import pytest
from fastapi.testclient import TestClient

from bee2bee_b200 import api as api_mod
from bee2bee_b200 import protocol as P
from bee2bee_b200.engine.core import Engine, SamplingParams
from bee2bee_b200.p2p_runtime import P2PNode
from bee2bee_b200.services import EmbeddedOllama, HFService

PROMPTS = [[1, 5, 9, 33, 2, 7], [4, 4, 19]]


def _record_submits(engine):
    """wrap ``engine.submit`` so every SamplingParams it receives is kept"""
    seen = []
    orig = engine.submit

    def submit(ids, params=None, on_token=None):
        seen.append(params)
        return orig(ids, params, on_token)

    engine.submit = submit
    return seen


def test_sampling_params_validation():
    eng = Engine("tiny-llama", device="cpu", max_batch=2, max_seq_len=64)
    for bad in (dict(top_k=-1), dict(min_p=-0.01), dict(min_p=1.5), dict(min_p=float("nan"))):
        with pytest.raises(ValueError):
            eng.submit([1, 2, 3], SamplingParams(max_new_tokens=2, **bad))
    assert SamplingParams().top_k == 0 and SamplingParams().min_p == 0.0
    out = eng.generate([[1, 2, 3]], SamplingParams(max_new_tokens=2, top_k=0, min_p=1.0, ignore_eos=True))
    assert len(out[0]) == 2


def test_top_k_beyond_int32_is_clamped_and_fails_no_request():
    """a top_k no int32 holds, submitted while another request runs: admission clamps it to the vocabulary (k >= V is
    off) and both requests finish"""
    eng = Engine("tiny-llama", device="cpu", max_batch=2, max_seq_len=64, decode_burst=2)
    admitted = []
    prefill = eng.runner.prefill

    def record(seqs):
        admitted.extend(seqs)
        return prefill(seqs)

    eng.runner.prefill = record
    r1 = eng.submit(PROMPTS[0], SamplingParams(max_new_tokens=8, ignore_eos=True))
    eng.step()
    assert not r1.done.is_set()
    r2 = eng.submit(PROMPTS[1], SamplingParams(max_new_tokens=8, ignore_eos=True, top_k=2 ** 31, seed=9))
    while not (r1.done.is_set() and r2.done.is_set()):
        eng.step()
    assert r1.error is None and r2.error is None
    assert len(r1.out_ids) == 8 and len(r2.out_ids) == 8
    assert [s.top_k for s in admitted] == [0, eng.cfg.vocab_size]


@pytest.mark.parametrize("filt", [dict(top_k=1), dict(min_p=1.0)])
def test_torch_runner_filter_reduces_to_greedy(filt):
    eng = Engine("tiny-llama", device="cpu", max_batch=2, max_seq_len=64)
    greedy = eng.generate(PROMPTS, SamplingParams(max_new_tokens=8, temperature=0.0, ignore_eos=True))
    sampled = eng.generate(PROMPTS, SamplingParams(max_new_tokens=8, temperature=0.8, ignore_eos=True, seed=5, **filt))
    plain = eng.generate(PROMPTS, SamplingParams(max_new_tokens=8, temperature=0.8, top_p=1.0, ignore_eos=True, seed=5))
    assert sampled == greedy
    assert plain != greedy


def test_ollama_options_reach_sampling_params():
    ol = EmbeddedOllama("tiny-llama", max_batch=2, max_seq_len=64, device="cpu")
    seen = _record_submits(ol._ensure().engine)
    list(ol.generate({"prompt": "hi", "stream": False, "options": {"num_predict": 2, "top_k": 7, "min_p": 0.05}}))
    list(ol.generate({"prompt": "hi", "stream": False, "options": {"num_predict": 2}}))
    # Ollama treats top_k <= 0 and min_p <= 0 as off: the request samples instead of failing
    out = list(ol.generate({"prompt": "hi", "stream": False, "options": {"num_predict": 2, "top_k": -1, "min_p": -0.5}}))
    assert out[-1]["done"] and out[-1]["eval_count"] == 2
    assert (seen[0].top_k, seen[0].min_p) == (7, 0.05)
    assert (seen[1].top_k, seen[1].min_p) == (0, 0.0)         # Ollama's own top_k default is not applied
    assert (seen[1].temperature, seen[1].top_p, seen[1].repetition_penalty) == (0.8, 0.9, 1.1)
    assert (seen[2].top_k, seen[2].min_p) == (0, 0.0)


def test_gen_request_without_filters_is_unchanged():
    base = {"type": "gen_request", "rid": "r", "prompt": "p", "model": "m", "svc": "hf", "max_new_tokens": 5,
            "max_tokens": 5, "temperature": 0.3, "stream": True}
    assert P.gen_request("r", "p", model="m", max_new_tokens=5, temperature=0.3, stream=True) == base
    assert list(P.gen_request("r", "p", model="m", max_new_tokens=5, temperature=0.3, stream=True)) == list(base)
    m = P.gen_request("r", "p", model="m", max_new_tokens=5, temperature=0.3, stream=True, top_k=9, min_p=0.1)
    assert m == {**base, "top_k": 9, "min_p": 0.1}
    assert P.gen_request("r", "p", top_k=3) == {**P.gen_request("r", "p"), "top_k": 3}


@pytest.fixture()
def client(monkeypatch):
    monkeypatch.setenv("BEE2BEE_TRANSPORT", "inproc")
    monkeypatch.delenv("BEE2BEE_API_KEY", raising=False)
    api_mod.node = None
    with TestClient(api_mod.app) as c:
        yield c
    api_mod.node = None


def test_generate_filters_reach_sampling_params_local(client):
    svc = HFService("tiny-llama", 0.0, max_batch=2, max_seq_len=128, device="cpu")
    svc.load_sync()
    api_mod.node.local_services["hf"] = svc
    seen = _record_submits(svc.model.engine)
    try:
        body = {"prompt": "user: hi", "max_new_tokens": 2, "temperature": 0.5}
        assert client.post("/generate", json={**body, "top_k": 12, "min_p": 0.25}).json()["status"] == "ok"
        assert client.post("/chat", json=body).json()["status"] == "ok"
        with client.stream("POST", "/generate", json={**body, "stream": True, "min_p": 0.5}) as resp:
            list(resp.iter_lines())
        assert client.post("/generate", json={**body, "top_k": -2}).json()["status"] == "error"
    finally:
        svc.model.engine.stop()
    assert [(s.top_k, s.min_p) for s in seen[:3]] == [(12, 0.25), (0, 0.0), (0, 0.5)]
    assert seen[0].top_p == 1.0 and seen[2].top_p == 0.95      # the paths' own defaults are unchanged


def test_generate_filters_reach_remote_provider(client, monkeypatch):
    calls = []

    async def fake_request_generation(pid, prompt, max_new_tokens=32, model_name=None, **kw):
        calls.append(kw)
        return {"text": "ok"}

    monkeypatch.setattr(api_mod.node, "request_generation", fake_request_generation)
    body = {"prompt": "x", "provider_id": "peer-elsewhere", "max_new_tokens": 3}
    assert client.post("/generate", json={**body, "top_k": 4, "min_p": 0.1}).json()["status"] == "ok"
    assert client.post("/generate", json=body).json()["status"] == "ok"
    assert calls[0] == {"temperature": 0.7, "top_k": 4, "min_p": 0.1}
    assert calls[1] == {"temperature": 0.7}


def test_mesh_requests_and_relay_carry_filters():
    """requester -> provider, requester -> relay -> provider, and a streamed request: the provider's engine receives
    the filters; a request without them reaches it with both off"""
    async def go():
        nodes = [P2PNode(host="127.0.0.1", port=0, transport="inproc", name=f"f{i}-{id(object())}",
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
            await a.request_generation(b.peer_id, "hello", 2, "tiny-llama", top_k=6, min_p=0.2, timeout=60)
            await a.request_generation(b.peer_id, "hello", 2, "tiny-llama", timeout=60)
            await a.request_generation(b.peer_id, "user: hi", 2, "tiny-llama", min_p=0.3, on_chunk=lambda s: None,
                                       timeout=60)
            # relay: c asks a, which does not serve the model and forwards to b
            await c._drop_peer(b.peer_id)
            c.providers.pop(b.peer_id, None)
            fut = asyncio.get_running_loop().create_future()
            c._pending_requests["r1"] = fut
            await c._send(c._conn_of(a.peer_id), P.gen_request("r1", "relay", model="tiny-llama", max_new_tokens=2,
                                                                top_k=3))
            out = await asyncio.wait_for(fut, 60)
            assert not out.get("error"), out
        finally:
            svc.model.engine.stop()
            for n in nodes:
                await n.stop()
        return seen

    seen = asyncio.run(go())
    assert [(s.top_k, s.min_p) for s in seen] == [(6, 0.2), (0, 0.0), (0, 0.3), (3, 0.0)]
