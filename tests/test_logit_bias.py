"""``logit_bias`` from the request surfaces down to the sampler's reference (CPU): parsing and refusals, the reference
sampler against a hand-written numpy one, the CPU engine and the CPU mesh pipeline, /generate and /chat (local and
relayed), the mesh ``gen_request`` message and relay, the supervised engine's JSON pipe and the multi-rank plan."""
import asyncio
import pickle

import numpy as np
import pytest
import torch
from fastapi.testclient import TestClient

from bee2bee_b200 import api as api_mod
from bee2bee_b200 import protocol as P
from bee2bee_b200.engine.core import LOGIT_BIAS_MAX, Engine, SamplingParams, parse_logit_bias
from bee2bee_b200.models.torch_ref import sample_reference
from bee2bee_b200.p2p_runtime import P2PNode
from bee2bee_b200.services import EmbeddedOllama, HFService, sampling_filters

PROMPT = [1, 5, 9, 33, 2, 7]


def _record_submits(engine):
    """wrap ``engine.submit`` so every SamplingParams it receives is kept"""
    seen = []
    orig = engine.submit

    def submit(ids, params=None, on_token=None):
        seen.append(params)
        return orig(ids, params, on_token)

    engine.submit = submit
    return seen


def _greedy(**kw):
    return SamplingParams(max_new_tokens=6, temperature=0.0, top_p=1.0, repetition_penalty=1.0, ignore_eos=True, **kw)


# --------------------------------------------------------------------------- parsing and refusals
def test_parse_logit_bias_takes_decimal_keys():
    assert parse_logit_bias(None) == {} and parse_logit_bias({}) == {}
    assert parse_logit_bias({"5": 1, "0": -100.0, "+7": 2.5, 9: 0.5}) == {5: 1.0, 0: -100.0, 7: 2.5, 9: 0.5}
    assert all(type(k) is int for k in parse_logit_bias({"5": 1, np.int64(6): 2}))
    for bad in ({"a": 1.0}, {"1.5": 1.0}, {"": 1.0}, {" 5": 1.0}, {"5_0": 1.0}, {"0x10": 1.0}, {True: 1.0},
                {2.0: 1.0}, {"5": "1"}, {"5": None}, {"5": True}, {"5": 1.0, "05": 2.0}, {"7": 1.0, 7: 1.0},
                [(5, 1.0)], "5"):
        with pytest.raises(ValueError):
            parse_logit_bias(bad)


def test_submit_refuses_bad_logit_bias():
    eng = Engine("tiny-llama", device="cpu", max_batch=2, max_seq_len=64)
    V = eng.cfg.vocab_size
    bad = [{V: 1.0}, {V + 100: 1.0}, {-1: 1.0}, {"5": 1.0}, {5.0: 1.0}, {3: float("nan")}, {3: float("inf")},
           {3: -float("inf")}, {3: 100.5}, {3: -100.01}, {3: "1"}, {i: 0.1 for i in range(LOGIT_BIAS_MAX + 1)}]
    for lb in bad:
        with pytest.raises(ValueError):
            eng.submit(PROMPT, _greedy(logit_bias=lb))
    assert SamplingParams().logit_bias == {}
    ok = {i: 0.0 for i in range(min(V, LOGIT_BIAS_MAX) - 1)}
    ok.update({V - 1: 100.0})
    SamplingParams(logit_bias={i: 1.0 for i in range(LOGIT_BIAS_MAX)}).validate(2 * LOGIT_BIAS_MAX)
    assert eng.generate([PROMPT], _greedy(logit_bias=ok))[0] == [V - 1] * 6
    assert eng.generate([PROMPT], _greedy(logit_bias={0: -100.0, 3: 100}))[0] == [3] * 6


def test_sampling_filters_carries_logit_bias_only_when_set():
    assert sampling_filters({"logit_bias": None}) == {} and sampling_filters({"logit_bias": {}}) == {}
    assert sampling_filters({"logit_bias": {"12": -3}, "top_k": 2}) == {"top_k": 2, "logit_bias": {12: -3.0}}
    with pytest.raises(ValueError):
        sampling_filters({"logit_bias": {"x": 1.0}})


# --------------------------------------------------------------------------- reference sampler
def _numpy_sample(raw, seen, counts, bias, temp, pen, pres, freq):
    """greedy / the post-temperature logits, step by step in float32: bias, repetition penalty, presence / frequency"""
    l = raw.astype(np.float32).copy()
    for t, b in bias.items():
        l[t] = np.float32(l[t] + np.float32(b))
    pl = np.where(l > 0, l / np.float32(pen), l * np.float32(pen)).astype(np.float32)
    l = np.where(seen, pl, l) if pen != 1.0 else l
    step = ((l - np.float32(freq) * counts.astype(np.float32)).astype(np.float32) - np.float32(pres)).astype(np.float32)
    l = np.where(counts > 0, step, l) if (pres or freq) else l
    return l if temp <= 0 else (l / np.float32(temp)).astype(np.float32)


def _bias_arg(bias):
    return (torch.tensor(list(bias), dtype=torch.long), torch.tensor(list(bias.values()), dtype=torch.float32))


def test_sample_reference_adds_bias_before_the_penalties():
    rng = np.random.default_rng(0)
    V = 500
    for i in range(16):
        raw = (rng.standard_normal(V) * 3).astype(np.float32)
        seen = rng.random(V) < 0.15
        counts = np.where(rng.random(V) < 0.2, rng.integers(1, 9, V), 0).astype(np.int32)
        ids = rng.choice(V, 30, replace=False)
        bias = {int(t): float(v) for t, v in zip(ids, rng.uniform(-6, 6, 30))}
        bias[int(np.argmax(raw))] = (-100.0, 100.0)[i % 2]
        pen, pres, freq = (1.0, 1.3)[i % 2], (0.0, 0.5)[(i // 2) % 2], (0.0, 0.25)[(i // 4) % 2]
        want = _numpy_sample(raw, seen, counts, bias, 0.0, pen, pres, freq)
        got = sample_reference(torch.from_numpy(raw)[None], torch.from_numpy(seen)[None], 0.0, 1.0, pen,
                               counts=torch.from_numpy(counts)[None], presence=pres, frequency=freq,
                               bias=_bias_arg(bias))
        assert int(got) == int(np.argmax(want)), i
        # sampled: the draws come from the softmax of the same float32 row (top_k = 1 keeps its argmax)
        got = sample_reference(torch.from_numpy(raw)[None], torch.from_numpy(seen)[None], 0.8, 1.0, pen,
                               torch.Generator().manual_seed(i), top_k=1, counts=torch.from_numpy(counts)[None],
                               presence=pres, frequency=freq, bias=_bias_arg(bias))
        assert int(got) == int(np.argmax(_numpy_sample(raw, seen, counts, bias, 0.8, pen, pres, freq))), i
    # the repetition penalty's sign test sees the biased logit: -1 + 2.5 = 1.5 > 0, so 1.5 / 2 = 0.75 beats 0.6
    raw = np.full(V, -5.0, np.float32)
    raw[10], raw[20] = -1.0, 0.6
    seen = np.zeros(V, bool)
    seen[10] = True
    args = (torch.from_numpy(raw)[None], torch.from_numpy(seen)[None], 0.0, 1.0, 2.0)
    assert int(sample_reference(*args)) == 20
    assert int(sample_reference(*args, bias=_bias_arg({10: 2.5}))) == 10
    raw[20] = 1.0
    assert int(sample_reference(*args, bias=_bias_arg({10: 2.5}))) == 20
    # only the listed ids move; an empty bias is no bias
    lg = torch.from_numpy((rng.standard_normal((3, V)) * 2).astype(np.float32))
    a = sample_reference(lg, None, 0.8, 0.9, 1.0, torch.Generator().manual_seed(1))
    b = sample_reference(lg, None, 0.8, 0.9, 1.0, torch.Generator().manual_seed(1), bias=_bias_arg({}))
    assert torch.equal(a, b)


# --------------------------------------------------------------------------- CPU backends
def test_cpu_engine_honours_bias_per_sequence():
    eng = Engine("tiny-llama", device="cpu", max_batch=2, max_seq_len=64)
    plain = eng.generate([PROMPT], _greedy())[0]
    g = plain[0]
    banned = eng.generate([PROMPT], _greedy(logit_bias={g: -100.0}))[0]
    assert banned[0] != g and g not in banned
    # a biased request beside a plain one, then the plain prompt again in the freed slots
    reqs = [eng.submit(PROMPT, _greedy(logit_bias={42: 100.0})), eng.submit(PROMPT, _greedy())]
    while not all(r.done.is_set() for r in reqs):
        eng.step()
    assert reqs[0].out_ids == [42] * 6 and reqs[1].out_ids == plain
    assert eng.generate([PROMPT, PROMPT], _greedy()) == [plain, plain]


def test_cpu_pipeline_honours_bias():
    from bee2bee_b200.parallel.cpu_pipeline import MeshPipelineService

    async def go():
        node = P2PNode(host="127.0.0.1", port=0, transport="inproc", name=f"lb-{id(object())}")
        await node.start()
        try:
            svc = MeshPipelineService(node, "tiny-llama", 1, [])
            svc.bind_loop(asyncio.get_running_loop())
            plain = await svc.agenerate(PROMPT, 5, temperature=0.0)
            forced = await svc.agenerate(PROMPT, 5, temperature=0.0, logit_bias={77: 100.0})
            banned = await svc.agenerate(PROMPT, 5, temperature=0.0, logit_bias={plain[0]: -100.0})
            with pytest.raises(ValueError):
                await svc.agenerate(PROMPT, 5, temperature=0.0, logit_bias={svc.cfg.vocab_size: 1.0})
            res = await svc.aexecute({"prompt": "hello", "max_new_tokens": 3, "temperature": 0.0,
                                      "logit_bias": {"77": 100}})
            return plain, forced, banned, res
        finally:
            await node.stop()

    plain, forced, banned, res = asyncio.run(go())
    assert forced == [77] * 5 and banned[0] != plain[0] and res["tokens"] == 3


# --------------------------------------------------------------------------- serving
def test_ollama_has_no_logit_bias():
    ol = EmbeddedOllama("tiny-llama", max_batch=2, max_seq_len=64, device="cpu")
    seen = _record_submits(ol._ensure().engine)
    list(ol.generate({"prompt": "hi", "stream": False, "options": {"num_predict": 2, "logit_bias": {"5": 100}}}))
    assert seen[0].logit_bias == {}
    from bee2bee_b200.services import OllamaService
    svc = OllamaService("tiny-llama", host="embedded")
    payload = svc._payload({"prompt": "x", "logit_bias": {"5": 1.0}, "top_k": 3}, stream=False)
    assert "logit_bias" not in payload["options"] and payload["options"]["top_k"] == 3


def test_gen_request_without_bias_is_unchanged():
    base = {"type": "gen_request", "rid": "r", "prompt": "p", "model": "m", "svc": "hf", "max_new_tokens": 5,
            "max_tokens": 5, "temperature": 0.3, "stream": True}
    for off in ({}, dict(logit_bias=None), dict(logit_bias={})):
        m = P.gen_request("r", "p", model="m", max_new_tokens=5, temperature=0.3, stream=True, **off)
        assert m == base and list(m) == list(base)
    m = P.gen_request("r", "p", model="m", max_new_tokens=5, temperature=0.3, stream=True, logit_bias={5: -1, 70: 2.5})
    assert m == {**base, "logit_bias": {"5": -1.0, "70": 2.5}}
    import json
    assert sampling_filters(json.loads(json.dumps(m))) == {"logit_bias": {5: -1.0, 70: 2.5}}


@pytest.fixture()
def client(monkeypatch):
    monkeypatch.setenv("BEE2BEE_TRANSPORT", "inproc")
    monkeypatch.delenv("BEE2BEE_API_KEY", raising=False)
    api_mod.node = None
    with TestClient(api_mod.app) as c:
        yield c
    api_mod.node = None


def test_generate_and_chat_bias_reaches_sampling_params_local(client):
    svc = HFService("tiny-llama", 0.0, max_batch=2, max_seq_len=128, device="cpu")
    svc.load_sync()
    api_mod.node.local_services["hf"] = svc
    seen = _record_submits(svc.model.engine)
    try:
        body = {"prompt": "user: hi", "max_new_tokens": 2, "temperature": 0.0}
        r = client.post("/generate", json={**body, "logit_bias": {"11": 100, "12": -5.5}}).json()
        assert r["status"] == "ok" and r["metadata"]["tokens"] == 2
        assert client.post("/chat", json={**body, "logit_bias": {}}).json()["status"] == "ok"
        assert client.post("/chat", json=body).json()["status"] == "ok"
        with client.stream("POST", "/generate", json={**body, "stream": True, "logit_bias": {"9": 3}}) as resp:
            list(resp.iter_lines())
        for bad in ({"x": 1}, {"5": 1, "05": 1}, {"5": 101}, {str(svc.model.engine.cfg.vocab_size): 1}):
            assert client.post("/generate", json={**body, "logit_bias": bad}).json()["status"] == "error", bad
    finally:
        svc.model.engine.stop()
    assert [s.logit_bias for s in seen[:4]] == [{11: 100.0, 12: -5.5}, {}, {}, {9: 3.0}]
    assert seen[0].top_p == 1.0 and seen[3].top_p == 0.95      # the paths' own defaults are unchanged


def test_generate_and_chat_bias_reaches_remote_provider(client, monkeypatch):
    calls = []

    async def fake_request_generation(pid, prompt, max_new_tokens=32, model_name=None, **kw):
        calls.append(kw)
        return {"text": "ok"}

    monkeypatch.setattr(api_mod.node, "request_generation", fake_request_generation)
    body = {"prompt": "x", "provider_id": "peer-elsewhere", "max_new_tokens": 3}
    assert client.post("/generate", json={**body, "logit_bias": {"3": 1.5}}).json()["status"] == "ok"
    assert client.post("/chat", json={**body, "logit_bias": {"4": -2}, "top_k": 2}).json()["status"] == "ok"
    assert client.post("/generate", json=body).json()["status"] == "ok"
    assert client.post("/generate", json={**body, "logit_bias": {"y": 1}}).json()["status"] == "error"
    assert calls == [{"temperature": 0.7, "logit_bias": {3: 1.5}}, {"temperature": 0.7, "top_k": 2,
                                                                     "logit_bias": {4: -2.0}}, {"temperature": 0.7}]


def test_mesh_requests_and_relay_carry_bias():
    """requester -> provider, requester -> relay -> provider, and a streamed request: the provider's engine receives
    the bias with int keys; a request without it reaches the provider with none; a malformed one is refused"""
    async def go():
        nodes = [P2PNode(host="127.0.0.1", port=0, transport="inproc", name=f"lb{i}-{id(object())}",
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
            await a.request_generation(b.peer_id, "hello", 2, "tiny-llama", logit_bias={7: 100.0}, timeout=60)
            await a.request_generation(b.peer_id, "hello", 2, "tiny-llama", timeout=60)
            await a.request_generation(b.peer_id, "user: hi", 2, "tiny-llama", logit_bias={8: -1},
                                       on_chunk=lambda s: None, timeout=60)
            # relay: c asks a, which does not serve the model and forwards to b
            await c._drop_peer(b.peer_id)
            c.providers.pop(b.peer_id, None)
            fut = asyncio.get_running_loop().create_future()
            c._pending_requests["r1"] = fut
            await c._send(c._conn_of(a.peer_id), P.gen_request("r1", "relay", model="tiny-llama", max_new_tokens=2,
                                                                logit_bias={9: 2.0}))
            out = await asyncio.wait_for(fut, 60)
            assert not out.get("error"), out
            fut = asyncio.get_running_loop().create_future()
            c._pending_requests["r2"] = fut
            msg = P.gen_request("r2", "relay", model="tiny-llama", max_new_tokens=2)
            msg["logit_bias"] = {"nine": 2.0}
            await c._send(c._conn_of(a.peer_id), msg)
            refused = await asyncio.wait_for(fut, 60)
        finally:
            svc.model.engine.stop()
            for n in nodes:
                await n.stop()
        return seen, refused

    seen, refused = asyncio.run(go())
    assert [s.logit_bias for s in seen] == [{7: 100.0}, {}, {8: -1.0}, {9: 2.0}]
    assert "logit_bias" in str(refused.get("error"))


@pytest.mark.timeout(600)
def test_supervised_engine_restores_int_keys():
    """the supervised engine's JSON pipe turns the int keys into strings: the worker restores them, so the bias acts;
    a bad id is refused in the caller, as by an in-process engine"""
    from bee2bee_b200.parallel.supervisor import SupervisedEngine
    sup = SupervisedEngine("tiny-llama", device="cpu", world=1, engine_kw=dict(max_batch=2, max_seq_len=256))
    try:
        assert sup.generate([PROMPT], _greedy(logit_bias={33: 100.0}))[0] == [33] * 6
        with pytest.raises(ValueError):
            sup.submit(PROMPT, _greedy(logit_bias={sup.cfg.vocab_size: 1.0}))
        assert sup.healthy and sup.restarts == 0
    finally:
        sup.close()


def test_plan_broadcast_keeps_the_bias():
    """the multi-rank plan travels through ``broadcast_object_list`` (pickle): a follower's mirror request has the
    same int-keyed bias"""
    import torch.distributed as dist
    eng = Engine("tiny-llama", device="cpu", max_batch=2, max_seq_len=64)
    r = eng.submit(PROMPT, _greedy(logit_bias={5: -100.0, 6: 2.5}))
    sent = []

    def broadcast(box, src=0, group=None):
        if eng.rank == 0:
            sent.append(pickle.dumps(box))
        else:
            box[0] = pickle.loads(sent[0])[0]

    orig = dist.broadcast_object_list
    dist.broadcast_object_list = broadcast
    try:
        eng.rank = 0
        eng._sync_plan([r])
        eng.rank = 1
        mirror = eng._sync_plan([])
    finally:
        dist.broadcast_object_list = orig
    assert len(mirror) == 1 and mirror[0].params.logit_bias == {5: -100.0, 6: 2.5}
    assert all(type(k) is int for k in mirror[0].params.logit_bias)
