"""World-size-2 gloo test of the cloud-key broadcast with a multi-bit bootstrap key (nufhe_b200.sharding:
broadcast_cloud_key): the receiver allocates a key of the sender's kind and ends up with the same key."""
import os
import socket

import torch
import torch.distributed as dist
import torch.multiprocessing as mp


def _worker(rank, world, port, results):
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import nufhe_b200 as nufhe
    from fake_engine import FakeEngine
    from nufhe_b200.sharding import broadcast_cloud_key
    dist.init_process_group('gloo', rank=rank, world_size=world)
    try:
        ctx = nufhe.Context(rng=nufhe.DeterministicRNG(91), thread=FakeEngine())
        sk = ctx.make_secret_key()
        params = sk.params
        ok = True
        for multi_bit in (2, 1):
            want = ctx.make_cloud_key(sk, multi_bit=multi_bit)        # every rank draws the same key from the seed
            got = broadcast_cloud_key(ctx.thread, params, want if rank == 0 else None, src=0)
            from nufhe_b200.sharding import cloud_key_tensors
            ok = ok and type(got.bootstrap_key) is type(want.bootstrap_key) and got.bootstrap_key.tgsw.shape == \
                want.bootstrap_key.tgsw.shape
            ok = ok and all(torch.equal(a, b) for a, b in zip(cloud_key_tensors(got), cloud_key_tensors(want)))
        results[rank] = bool(ok)
    finally:
        dist.destroy_process_group()


def test_broadcast_multibit_cloud_key_world_size_2():
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        port = s.getsockname()[1]
    ctx = mp.get_context('spawn')
    with ctx.Manager() as manager:
        results = manager.dict()
        procs = [ctx.Process(target=_worker, args=(r, 2, port, results)) for r in range(2)]
        for p in procs:
            p.start()
        for p in procs:
            p.join(600)
        assert all(p.exitcode == 0 for p in procs)
        assert dict(results) == {0: True, 1: True}
