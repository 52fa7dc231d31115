"""L0/L1: utils, config, join links, byte pieces, DHT, registry, STUN/NAT (intent of the
reference's tests/test_utils.py, test_p2p.py, test_pieces2.py, test_dht.py, test_nat_optional.py)."""
import asyncio
import json
import os
import socket
import struct

import pytest

from bee2bee_b200 import config, dht, nat, p2p, pieces, registry, stun_client, utils


def test_ids_and_hashing():
    a, b = utils.new_id("peer"), utils.new_id("peer")
    assert a != b and a.startswith("peer-") and len(a) == len("peer-") + 8
    assert utils.sha256_hex("x") == utils.sha256_hex("x") and len(utils.sha256_hex("x")) == 64
    s = utils.gen_salt()
    assert utils.hash_password("pw", s) == utils.hash_password("pw", s) != utils.hash_password("pw2", s)
    assert abs(utils.now_ms() - __import__("time").time() * 1000) < 5000


def test_home_and_atomic_json(tmp_path):
    home = utils.bee2bee_home()
    assert str(home) == os.environ["BEE2BEE_HOME"] and home.exists()
    f = utils.data_file("sub/x.json")
    utils.save_json(f, {"a": [1, 2]})
    assert utils.load_json(f, None) == {"a": [1, 2]}
    assert utils.load_json(home / "missing.json", 7) == 7
    f.write_text("{broken")
    assert utils.load_json(f, "dflt") == "dflt"
    assert not list(f.parent.glob("*.tmp"))


def test_system_metrics_keys_and_measured_throughput():
    m = utils.get_system_metrics()
    assert set(m) == {"throughput", "memory_percent", "gpu_percent", "trust_score"}
    utils.set_throughput_source(lambda: 1234.56)
    try:
        assert utils.get_system_metrics()["throughput"] == 1234.6
    finally:
        utils.set_throughput_source(None)
    assert isinstance(utils.get_gpu_usage(), float)      # multi-line nvidia-smi output must not raise


def test_config_tiers(monkeypatch):
    assert config.load_config()["bootstrap_url"] == "ws://127.0.0.1:4003"
    assert config.load_config()["api_port"] == 4002 and config.load_config()["p2p_port"] == 0
    config.set_bootstrap_url("ws://10.0.0.1:1")
    assert config.get_bootstrap_url() == "ws://10.0.0.1:1"
    monkeypatch.setenv("BEE2BEE_BOOTSTRAP", "ws://env:2")
    assert config.get_bootstrap_url() == "ws://env:2"
    config.save_config({"api_port": "not-a-number", "max_batch": "16", "custom": 1})
    cfg = config.load_config()
    assert cfg["api_port"] == 4002 and cfg["max_batch"] == 16 and cfg["custom"] == 1
    monkeypatch.setenv("BEE2BEE_PIECES", "8")
    assert config.get_setting("pieces") == 8


def test_join_link_roundtrip_and_schemes():
    link = p2p.generate_join_link("net", "distilgpt2", "abc123", ["ws://127.0.0.1:4003", "ws://h:9/x?y=1"])
    assert link.startswith("coithub.org://join?network=net&model=distilgpt2&hash=abc123&bootstrap=")
    assert "=" not in link.split("bootstrap=", 1)[1].split("&")[0]          # unpadded url-safe base64
    d = p2p.parse_join_link(link)
    assert d == {"network": "net", "model": "distilgpt2", "hash": "abc123",
                 "bootstrap": ["ws://127.0.0.1:4003", "ws://h:9/x?y=1"]}
    for scheme in ("coithub", "p2pnet"):
        assert p2p.parse_join_link(link.replace("coithub.org", scheme, 1))["bootstrap"][0] == "ws://127.0.0.1:4003"
    with pytest.raises(ValueError):
        p2p.parse_join_link("http://join?network=x")
    with pytest.raises(ValueError):
        p2p.parse_join_link("coithub.org://other?network=x")
    url = p2p.registration_url(link, "US-West", "hf", 8000)
    assert url.startswith("https://coithub.org/register?link=coithub.org%3A%2F%2Fjoin") and "api_port=8000" in url
    assert p2p.bitfield_from_pieces(5, [0, 3, 9, -1]) == [1, 0, 0, 1, 0]


def test_byte_pieces_roundtrip(tmp_path):
    data = b"Hello World" * 100
    chunks = pieces.split_pieces(data, 32)
    hashes = pieces.piece_hashes(chunks)
    assert len(chunks) == (len(data) + 31) // 32 and pieces.verify_and_reassemble(chunks, hashes) == data
    bad = list(chunks)
    bad[3] = b"x" * 32
    with pytest.raises(ValueError, match="hash_mismatch_at_3"):
        pieces.verify_and_reassemble(bad, hashes)
    with pytest.raises(ValueError, match="length_mismatch"):
        pieces.verify_and_reassemble(chunks[:-1], hashes)
    h = p2p.sha256_hex_bytes(data)
    paths = pieces.save_pieces(str(tmp_path), h, chunks)
    assert os.path.basename(paths[1]) == f"{h}_00000001.part"
    assert b"".join(pieces.load_pieces(str(tmp_path), h)) == data


def test_layer_piece_plan_and_checkpoint(tmp_path):
    import torch

    plan = pieces.plan_pieces("gemma-2-2b", 26, 4)
    assert [(p.start, p.end) for p in plan] == [(0, 7), (7, 14), (14, 20), (20, 26)]
    assert plan[0].first and plan[-1].last and not plan[1].first and plan[2].device == "cuda:2"
    tensors = {"l7.wq": torch.randn(8, 8), "l7.wo": torch.randn(8, 8).to(torch.bfloat16)}
    man = pieces.save_piece_checkpoint(str(tmp_path), plan[1], tensors, piece_size=100)
    back = pieces.load_piece_checkpoint(man)
    assert torch.equal(back["l7.wq"], tensors["l7.wq"]) and torch.equal(back["l7.wo"], tensors["l7.wo"])
    # corrupt one part file -> verification fails on resume
    part = sorted(p for p in os.listdir(tmp_path) if p.endswith(".part"))[0]
    with open(tmp_path / part, "r+b") as fh:
        fh.write(b"\xff\xff")
    with pytest.raises(ValueError):
        pieces.load_piece_checkpoint(man)


def test_dht_in_memory_and_mesh_local():
    async def go():
        node = dht.DHTNode()
        await node.start()
        assert isinstance(node.backend, dht.InMemoryDHT)        # kademlia absent / offline -> fake backend
        await dht.announce_piece(node, "abc", "ws://a:1")
        await dht.announce_piece(node, "abc", "ws://a:1")
        await dht.announce_piece(node, "abc", "ws://b:2")
        assert await dht.find_providers(node, "abc") == ["ws://a:1", "ws://b:2"]
        assert await dht.find_providers(node, "zzz") == []
        dht.MeshDHT.reset()
        m1, m2 = dht.DHTNode(mesh_local=True), dht.DHTNode(mesh_local=True)
        await m1.start(); await m2.start()
        await dht.announce_piece(m1, "k", "inproc://x")
        assert await dht.find_providers(m2, "k") == ["inproc://x"]     # one table per box

    asyncio.run(go())


def test_registry_offline_mode_and_payload(monkeypatch):
    for k in ("SUPABASE_URL", "VITE_SUPABASE_URL", "SUPABASE_ANON_KEY", "VITE_SUPABASE_ANON_KEY", "BEE2BEE_ENTRYPOINT"):
        monkeypatch.delenv(k, raising=False)
    reg = registry.RegistryClient()
    assert not reg.enabled
    ok = asyncio.run(reg.sync_node("peer-1", "ws://x:1", ["m"], tag="cli-net", region="EU", metrics={"a": 1}))
    assert ok is False
    row = registry.RegistryClient.local_rows()["peer-1"]
    assert set(row) == {"peer_id", "addr", "models", "latency_ms", "region", "tag", "metrics", "last_seen"}
    monkeypatch.setenv("SUPABASE_URL", "https://proj.supabase.co/")
    monkeypatch.setenv("SUPABASE_ANON_KEY", "key")
    reg = registry.RegistryClient()
    assert reg.enabled and reg.api_url == "https://proj.supabase.co/rest/v1/active_nodes"
    assert reg.headers["Prefer"] == "resolution=merge-duplicates" and reg.headers["apikey"] == "key"
    monkeypatch.delenv("SUPABASE_URL"); monkeypatch.delenv("SUPABASE_ANON_KEY")
    reg = registry.RegistryClient(entrypoint_url="http://entry:9/")
    assert reg.api_url == "http://entry:9/api/nodes/register"


def test_stun_message_codec():
    c = stun_client.STUNClient()
    req = c.create_binding_request()
    mtype, mlen, cookie = struct.unpack("!HHI", req[:8])
    assert (mtype, mlen, cookie, len(req)) == (0x0001, 0, 0x2112A442, 20)
    port = 40000 ^ (0x2112A442 >> 16)
    addr = struct.unpack("!I", socket.inet_aton("203.0.113.9"))[0] ^ 0x2112A442
    attr = struct.pack("!HHBBHI", 0x0020, 8, 0, 1, port, addr)
    resp = struct.pack("!HHI", 0x0101, len(attr), 0x2112A442) + req[8:] + attr
    assert c.parse_binding_response(resp) == {"ip": "203.0.113.9", "port": 40000, "xor": True}
    assert c.parse_binding_response(resp[:10]) is None
    assert c.parse_binding_response(struct.pack("!HHI", 0x0101, 0, 0x2112A442) + b"\0" * 12) is None   # wrong txid


def test_nat_api_is_inert_offline():
    async def go():
        ok, ip = await nat.try_upnp_map(4001)          # awaited (the reference test forgets to)
        assert ok is False and ip is None
        assert await nat.try_stun() is None
        assert await nat.get_public_ip() is None
        res = await nat.auto_port_forward(4001)
        assert isinstance(res, nat.PortForwardingResult) and not res and "offline" in str(res)

    asyncio.run(go())
    r = nat.PortForwardingResult(True, "UPnP", "1.2.3.4", 4001)
    assert bool(r) and str(r) == "UPnP: 1.2.3.4:4001"
    assert nat.PortForwarder()._is_valid_ip("10.0.0.1") and not nat.PortForwarder()._is_valid_ip("nope")


def test_mesh_staging_plan_sizes_quantised_hop_buffers():
    """fp8 across the handoff: the hop slots for the e4m3 stream, its scale-factor chunks (chunk layout: 512 B per
    32-row tile and 128 K) and the sum-of-squares counters exist only for mxfp8 meshes; a gate/up | down cut adds the
    e4m3 MLP hidden.  (Pure sizing logic -- the buffers themselves are cudaMalloc + IPC, tests/test_multigpu.py.)"""
    import torch
    from bee2bee_b200.parallel.mesh import MeshComm
    m = MeshComm(0, 1, torch.device("cpu"), hidden=4096, max_tokens=512, groups=8, group_batch=32, hist_len=256)
    assert not any(k in m._sizes() for k in ("stage_q", "stage_sf", "stage_ss", "stage_qh"))      # bf16 mesh: bf16 slots only
    m = MeshComm(0, 1, torch.device("cpu"), hidden=4096, max_tokens=512, groups=8, group_batch=32, hist_len=256,
                 ffn=14336, mx=True)
    s = m._sizes()
    assert s["stage_q"] == 8 * 32 * 4096 and s["stage_q_pf"] == 2 * 512 * 4096
    assert s["stage_sf"] == 8 * (1 * 32 * 512) and s["stage_sf_pf"] == 2 * (16 * 32 * 512)
    assert s["stage_ss"] == 8 * 32 * 4 and s["stage_ss_pf"] == 2 * 512 * 4
    assert s["stage_qh"] == 8 * 32 * 14336 and s["stage_sfh_pf"] == 2 * (16 * 112 * 512)
    assert all(v % 16 == 0 for k, v in s.items() if k.startswith("stage_sf")), "cp.async.bulk needs 16-byte aligned slots"
    # a single-rank mesh has no endpoints at all
    assert m.handoff(0).in_q == 0 and m.handoff_prefill(1).out_q == 0
