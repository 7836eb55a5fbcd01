"""Multi-GPU plumbing: ciphertext batches shard on the leading axis; the cloud key is broadcast once.

The reference's only multi-GPU model is "one Context per device, keys and ciphertext slices moved as
pickled bytes through the host" (examples/multi_gpu.py:46-104).  Here one process drives one GPU
(`torch.distributed`, NCCL over NVLink on the box, gloo in the CPU tests); there is no per-gate
collective because ciphertexts are independent (SURVEY.md section 8e)."""
import torch
import torch.distributed as dist


def shard_bounds(batch, world, rank):
    """Contiguous, balanced split of `batch` items: ranks < batch % world get one extra item."""
    base, extra = divmod(batch, world)
    start = rank * base + min(rank, extra)
    return start, start + base + (1 if rank < extra else 0)


def cloud_key_tensors(cloud_key):
    """The device arrays that make up a NuFHECloudKey, in a fixed order."""
    ks = cloud_key.keyswitch_key.lwe
    return [cloud_key.bootstrap_key.tgsw.samples.a.coeffs, ks.a, ks.b, ks.current_variances]


def empty_cloud_key(thr, params, multi_bit=1):
    """A cloud key of the given kind with allocated, unfilled arrays: what a receiving rank broadcasts into.
    multi_bit=2 gives a MultiBitBootstrapKey (3n/2 rows), 1 a BootstrapKey (n rows)."""
    from .api_low_level import NuFHECloudKey
    from .bootstrap import BootstrapKey, MultiBitBootstrapKey, MultiBitTGswSampleArray, check_multi_bit
    from .lwe import LweKeyswitchKey, LweSampleArray
    from .tgsw import TransformedTGswSampleArray
    check_multi_bit(params, multi_bit)
    n = params.in_out_params.size
    rows = 3 * n // 2 if multi_bit == 2 else n
    tg_cls, bk_cls = ((MultiBitTGswSampleArray, MultiBitBootstrapKey) if multi_bit == 2
                      else (TransformedTGswSampleArray, BootstrapKey))
    tg = tg_cls.empty(thr, params.tgsw_params, (rows,))
    tl = params.tgsw_params.tlwe_params
    in_size = tl.mask_size * tl.polynomial_degree
    ks = LweSampleArray.empty(thr, params.in_out_params, (in_size, params.ks_decomp_length, 2**params.ks_log2_base))
    return NuFHECloudKey(params, bk_cls(params.in_out_params, tg), LweKeyswitchKey(ks))


def broadcast_cloud_key(thr, params, cloud_key=None, src=0, group=None):
    """The cloud key of rank `src` on every rank: `src` passes its key, the others None.  The key kind (standard or
    multi-bit) is broadcast first, so that every receiver allocates a key of the sender's kind; returns the key."""
    kind = torch.tensor([getattr(cloud_key.bootstrap_key, 'multi_bit', 1) if cloud_key is not None else 0],
                        dtype=torch.int64, device=thr.device)
    dist.broadcast(kind, src=src, group=group)
    if dist.get_rank(group) != src:
        cloud_key = empty_cloud_key(thr, params, int(kind.item()))
    broadcast_tensors(cloud_key_tensors(cloud_key), src=src, group=group)
    return cloud_key


def broadcast_tensors(tensors, src=0, group=None):
    """Broadcast each tensor from `src` in place (one collective per tensor, set-up time only)."""
    for t in tensors:
        dist.broadcast(t, src=src, group=group)


def gather_shards(local, batch, world, rank, group=None):
    """All-gather variable-size leading-axis shards back into the full batch (host-side convenience for
    examples and tests; the benchmark never gathers inside the timed region)."""
    sizes = [shard_bounds(batch, world, r) for r in range(world)]
    maxlen = max(e - s for s, e in sizes)
    pad = torch.zeros((maxlen,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    pad[:local.shape[0]] = local
    out = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(out, pad, group=group)
    return torch.cat([o[:e - s] for o, (s, e) in zip(out, sizes)], dim=0)
