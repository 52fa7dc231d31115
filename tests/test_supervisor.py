"""Dead-worker recovery (SURVEY 5.3, VERDICT r1 missing #5): the serving front keeps running in its own process, the engine
group is a child that can be killed; in-flight requests fail at once, the provider reports unhealthy while the group is
down, a fresh group comes up and serves again.  CPU worker here; on a GPU box the same supervisor spawns one worker
per GPU piece (a dead rank cannot be repaired inside the process that shares its CUDA context)."""
import os
import signal
import time

import pytest

from bee2bee_b200.engine.core import SamplingParams
from bee2bee_b200.parallel.supervisor import SupervisedEngine


@pytest.mark.timeout(900)
def test_supervised_engine_survives_a_killed_worker():
    sup = SupervisedEngine("tiny-llama", device="cpu", world=1, engine_kw=dict(max_batch=2, max_seq_len=2048))
    try:
        sp = SamplingParams(max_new_tokens=5, temperature=0.0, ignore_eos=True)
        first = sup.generate([[1, 2, 3], [4, 5]], sp)
        assert [len(o) for o in first] == [5, 5] and sup.healthy and sup.restarts == 0
        # streaming: tokens arrive one by one through the control channel, in order
        got = []
        r = sup.submit([1, 2, 3], sp, on_token=got.append)
        r.wait(timeout=60)
        assert got == first[0] == r.out_ids and r.finish_reason == "length" and r.ttft_ms > 0
        m = sup.metrics()
        assert m["supervised"] and m["requests"] >= 3 and m["healthy"]
        # cancellation crosses the channel
        long = sup.submit([7, 8, 9], SamplingParams(max_new_tokens=1500, temperature=0.0, ignore_eos=True))
        time.sleep(0.3)
        sup.cancel(long)
        long.done.wait(30)
        assert long.finish_reason == "cancelled" and len(long.out_ids) < 1500
        # kill the worker under an in-flight request
        victim = sup.submit([7, 8, 9], SamplingParams(max_new_tokens=1500, temperature=0.0, ignore_eos=True))
        time.sleep(0.2)
        pid = sup.worker_pids()[0]
        os.kill(pid, signal.SIGKILL)                       # the exact pid the supervisor started
        assert victim.done.wait(30), "in-flight request was not failed"
        assert victim.error and "restarted" in victim.error
        with pytest.raises(RuntimeError):
            victim.wait()
        # while the group is down new work is refused at once (the mesh routes around an unhealthy provider)
        if not sup.healthy:
            refused = sup.submit([1], sp)
            assert refused.done.is_set() and refused.error
        assert sup.wait_healthy(120), sup.broken
        assert sup.restarts == 1 and sup.worker_pids()[0] != pid
        assert sup.generate([[1, 2, 3], [4, 5]], sp) == first          # same weights, same greedy tokens
    finally:
        sup.close()
    assert sup.broken == "closed" and not sup.worker_pids()


def test_hf_loader_can_put_the_engine_behind_the_supervisor(monkeypatch):
    from bee2bee_b200 import hf

    monkeypatch.setenv("B2B_SUPERVISED", "1")
    lm, tok, dev = hf.load_model_and_tokenizer("tiny-gpt2", device="cpu", max_batch=2, max_seq_len=128)
    try:
        assert type(lm.engine).__name__ == "SupervisedEngine" and lm.config.name
        text = hf.generate_text(lm, tok, dev, "hello", max_new_tokens=4, temperature=0.0)
        assert text.startswith("hello") and len(text) > len("hello")
        chunks = list(hf.generate_text_stream(lm, tok, dev, "user: hi", max_new_tokens=6, temperature=0.0))
        assert isinstance("".join(chunks), str)
    finally:
        hf.unload_model("tiny-gpt2")
