"""A CPU test double for the expansion of compressed cloud keys into multi-key slots (DESIGN.md section 19).  TEST
INFRASTRUCTURE ONLY.

The multi-key engine double of tests/multikey_ops_fake.py plus the three slot calls of nufhe_b200.engine.Engine: a slot
holds the bootstrap key in the double's layout (the transformed TGSW coefficients, what its bk_prepare returns), and
both expansions are composed per tenant from the steps of CompressedCloudKey.decompress(), so the machine on compressed
keys runs in the CPU suite against exactly what per-tenant VirtualMachines on decompressed keys compute.  Every
expansion is recorded in `expansions` as (kind, number of tenants)."""
import torch

from nufhe_b200.compressed import _bk_masks, _ks_masks
from nufhe_b200.tgsw import TGswSampleArray, TransformedTGswSampleArray, tgsw_transform_samples
from fake_engine import N
from multikey_ops_fake import MultiKeyOpsFakeEngine


class MultiKeyPoolFakeEngine(MultiKeyOpsFakeEngine):

    def __init__(self):
        super().__init__()
        self.expansions = []
        self._bk_cache, self._ks_cache = {}, {}

    def mk_bk_slot(self, n):
        return torch.zeros((n, 2, 2, 2, N), dtype=torch.int64)

    def mk_bk_expand(self, seeds, bodies, slots, params):
        assert len(seeds) == len(bodies) == len(slots)
        self.expansions.append(('bk', len(slots)))
        for seed, body, slot in zip(seeds, bodies, slots):
            key = (bytes(seed.astype('uint32')), body.data_ptr())
            if key not in self._bk_cache:
                bk_params = params.tgsw_params
                k = bk_params.tlwe_params.mask_size
                rows = body.shape[0]
                bk = TGswSampleArray.empty(self, bk_params, (rows,))
                coeffs = bk.samples.a.coeffs
                coeffs[..., :k, :] = _bk_masks(self, seed, bk_params, rows)
                coeffs[..., k, :] = body
                out = TransformedTGswSampleArray.empty(self, bk_params, (rows,))
                tgsw_transform_samples(self, out, bk)
                self._bk_cache[key] = self.bk_prepare(out.samples.a.coeffs).clone()
            slot.copy_(self._bk_cache[key].reshape(slot.shape))

    def mk_ks_expand(self, seeds, ks_as):
        assert len(seeds) == len(ks_as)
        self.expansions.append(('ks', len(ks_as)))
        for seed, ks_a in zip(seeds, ks_as):
            in_size, t, base, n = ks_a.shape
            key = bytes(seed.astype('uint32'))
            if key not in self._ks_cache:
                self._ks_cache[key] = _ks_masks(self, seed, in_size, t, base, n)
            ks_a[:, :, 0, :] = 0
            ks_a[:, :, 1:, :] = self._ks_cache[key]
