"""A CPU test double for the multi-key calls of nufhe_b200.engine.Engine (nb_mk_*, DESIGN.md section 17).  TEST
INFRASTRUCTURE ONLY.

The engine double of tests/fake_engine.py plus the programmable bootstrap of tests/test_host_lut.py, with the four
multi-key methods composed per tenant from the single-key ones: tenant t owns counts[t] consecutive rows of the batch
and is served by the single-key method with its own key, so the Python layer of nufhe_b200/multikey.py runs in the CPU
suite against exactly what per-tenant VirtualMachines compute."""
import torch

from fake_engine import N
from test_host_lut import LutFakeEngine


class MultiKeyFakeEngine(LutFakeEngine):

    # --- the multi-key calls, composed per tenant from the single-key ones (tenant t owns counts[t] consecutive rows)
    @staticmethod
    def _segments(counts):
        lo = 0
        for t, cnt in enumerate(counts):
            yield t, lo, lo + int(cnt)
            lo += int(cnt)

    @staticmethod
    def _rows(x, lo, hi):
        if x is None:
            return None
        return x[0].reshape(-1, x[0].shape[-1])[lo:hi], x[1].reshape(-1)[lo:hi]

    @staticmethod
    def _cat(parts, width):
        if not parts:
            return torch.empty((0, width), dtype=torch.int32), torch.empty((0,), dtype=torch.int32)
        return torch.cat([p[0].reshape(-1, width) for p in parts]), torch.cat([p[1].reshape(-1) for p in parts])

    def mk_bootstrap_extract(self, x1, x2, c, s1, s2, mu, bk_ints, counts):
        assert len(bk_ints) == len(counts) and sum(counts) == x1[1].numel()
        return self._cat([self.bootstrap_extract(self._rows(x1, lo, hi), self._rows(x2, lo, hi), c, s1, s2, mu, bk_ints[t])
                          for t, lo, hi in self._segments(counts) if hi > lo], N)

    def mk_bootstrap_lut_extract(self, x1, x2, c, s1, s2, tv, log2_outputs, bk_ints, counts):
        assert len(bk_ints) == len(counts) and sum(counts) == x1[1].numel()
        return self._cat([self.bootstrap_lut_extract(self._rows(x1, lo, hi), self._rows(x2, lo, hi), c, s1, s2, tv,
                                                     log2_outputs, bk_ints[t])
                          for t, lo, hi in self._segments(counts) if hi > lo], N)

    def mk_bootstrap_extract2(self, job_a, job_b, mu, bk_ints, counts):
        def job(j, lo, hi):
            return (self._rows(j[0], lo, hi), self._rows(j[1], lo, hi)) + tuple(j[2:])
        assert len(bk_ints) == len(counts) and sum(counts) == job_a[0][1].numel()
        pairs = [self.bootstrap_extract2(job(job_a, lo, hi), job(job_b, lo, hi), mu, bk_ints[t])
                 for t, lo, hi in self._segments(counts) if hi > lo]
        return self._cat([p[0] for p in pairs], N), self._cat([p[1] for p in pairs], N)

    def mk_keyswitch(self, keys, counts, src1, src2=None, c=0, want_cv=False):
        assert len(keys) == len(counts) and sum(counts) == src1[1].numel()
        n = keys[0][0].shape[-1]
        parts = [self.keyswitch(keys[t], self._rows(src1, lo, hi), self._rows(src2, lo, hi), c, want_cv=True)
                 for t, lo, hi in self._segments(counts) if hi > lo]
        ra, rb = self._cat(parts, n)
        rcv = torch.cat([p[2].reshape(-1) for p in parts]) if parts else torch.empty((0,), dtype=torch.float32)
        return ra, rb, (rcv if want_cv else None)
