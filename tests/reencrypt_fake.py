"""A CPU test double for re-encryption (DESIGN.md section 22).  TEST INFRASTRUCTURE ONLY.

The multi-key engine double on compressed keys (tests/multikey_pool_fake.py, which has the compact, packing and
multi-key calls) plus Engine.reencrypt composed per segment from tests/reencrypt_ref.py.  The double's spectra are the
oracle's NTT, so each segment's mask is recovered with the oracle's inverse transform."""
import torch

from fake_engine import N, _np, _t
from multikey_pool_fake import MultiKeyPoolFakeEngine
import reencrypt_ref


class ReencryptFakeEngine(MultiKeyPoolFakeEngine):

    def reencrypt(self, a, b, spectra, bodies, counts):
        self._count('reencrypt')
        assert len(spectra) == len(bodies) == len(counts) and sum(counts) == b.numel() == a.shape[0]
        self.reencrypt_segments = getattr(self, 'reencrypt_segments', []) + [list(counts)]
        parts, lo = [], 0
        for spec, body, cnt in zip(spectra, bodies, counts):
            mask = _np(self.ntt_inverse_i32(spec)).reshape(-1)
            if cnt:
                parts.append(reencrypt_ref.reencrypt(_np(a[lo:lo + cnt]), _np(b[lo:lo + cnt]), mask, _np(body)))
            lo += cnt
        return (torch.cat([_t(p[0]) for p in parts]), torch.cat([_t(p[1]) for p in parts]))
