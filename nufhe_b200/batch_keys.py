"""The keys that serve the rows of a batch (DESIGN.md section 18): `OneKey` serves every row with one cloud key through
the single-key engine calls, `TenantKeys` a batch concatenated from several tenants through the multi-key calls.  Where
an item stands for several rows (a ciphertext's level-1 test vectors, a query's W columns), a call takes the rows per
item as `per`."""
import numpy

from .bootstrap import _single_kernel
from .tgsw import engine_format


def owners(counts, r0, r1):
    """The segments (counts[i] items each, in order) that own some of the items [r0, r1) of their concatenation, and
    how many they own."""
    hi = numpy.cumsum(counts, dtype=numpy.int64)
    own = numpy.clip(numpy.minimum(hi, r1) - numpy.maximum(hi - counts, r0), 0, None)
    idx = numpy.nonzero(own)[0]
    return idx, [int(own[i]) for i in idx]


def group_rows(counts, N, pad):
    """Slot s of the groups of N slots in which each segment (counts[i] rows, in order) starts a new group: row
    rows[s] of the concatenated rows, or `pad` in the slots that pad a segment's last group.  Returns (groups, rows)."""
    groups = [-(-c // N) for c in counts]
    rows = numpy.full(sum(groups) * N, pad, numpy.int64)
    g0 = c0 = 0
    for c, g in zip(counts, groups):
        rows[g0 * N:g0 * N + c] = numpy.arange(c0, c0 + c)
        g0, c0 = g0 + g, c0 + c
    return groups, rows


class OneKey:
    """One cloud key for every row: the bootstrap key `bk`, the LweKeyswitchKey `ks`, the tree key whose planes
    serve `tree_keyswitch` and the packing spectra (_GadgetKey.spectra) that serve `ntt_mac`, as far as the operation
    needs them.  The bootstraps run fused when perf_params and the key allow it, else as the reference's steps."""

    def __init__(self, thr, bk=None, ks=None, perf_params=None, tree_key=None, spectra=None):
        self.thr, self.bk, self.ks, self.perf_params = thr, bk, ks, perf_params
        self.tree_key, self.spectra = tree_key, spectra

    def split(self, r0, r1):
        return self

    def bootstrap_lut_extract(self, x1, x2, s1, tv, L, per=1):
        if _single_kernel(self.perf_params, self.bk):
            return self.thr.bootstrap_lut_extract(x1, x2, 0, s1, 1, tv, L, engine_format(self.thr, self.bk.tgsw))
        from .lut import _lut_steps
        return _lut_steps(self.thr, self.bk, x1, x2, s1, tv, L, x1[1].shape[0], self.perf_params)

    def bootstrap_glwe_lut_extract(self, x, tv, per=1):
        if _single_kernel(self.perf_params, self.bk):
            return self.thr.bootstrap_glwe_lut_extract(x, tv, engine_format(self.thr, self.bk.tgsw))
        from .tree_lut import _glwe_steps
        return _glwe_steps(self.thr, self.bk, x, tv, self.perf_params)

    def keyswitch(self, src, per=1, out=None, want_cv=False):
        return self.thr.keyswitch(self.ks.device_arrays(), src, out=out, want_cv=want_cv)

    def tree_keyswitch(self, a, mask_size, per=1):
        return self.thr.tree_keyswitch(a, self.tree_key.planes(self.thr), mask_size)

    def ntt_mac(self, x, per=1):
        return self.thr.ntt_mac(x, self.spectra)


class TenantKeys:
    """The keys of tenants whose items are concatenated in order, counts[i] items of the i-th: engine-format bootstrap
    keys `bks`, key-switch arrays `kss` (ks_a, ks_b, ks_cv), tree planes and packing spectra, as the operation needs."""

    def __init__(self, thr, counts, bks=None, kss=None, planes=None, spectra=None):
        self.thr, self.counts = thr, list(counts)
        self.bks, self.kss, self.planes, self.spectra = bks, kss, planes, spectra

    def split(self, r0, r1):
        """The keys of the items [r0, r1)."""
        idx, own = owners(self.counts, r0, r1)
        pick = lambda lst: None if lst is None else [lst[i] for i in idx]
        return TenantKeys(self.thr, own, pick(self.bks), pick(self.kss), pick(self.planes), pick(self.spectra))

    def _rows(self, per):
        return [c * per for c in self.counts]

    def bootstrap_lut_extract(self, x1, x2, s1, tv, L, per=1):
        return self.thr.mk_bootstrap_lut_extract(x1, x2, 0, s1, 1, tv, L, self.bks, self._rows(per))

    def bootstrap_glwe_lut_extract(self, x, tv, per=1):
        return self.thr.mk_bootstrap_glwe_lut_extract(x, tv, self.bks, self._rows(per))

    def keyswitch(self, src, per=1, out=None, want_cv=False):
        """The multi-key key switch; with `out` = (a, b), copied into it (the multi-key call writes its own arrays)."""
        ra, rb, rcv = self.thr.mk_keyswitch(self.kss, self._rows(per), src, want_cv=want_cv)
        if out is not None:
            ra, rb = out[0].copy_(ra), out[1].copy_(rb)
        return ra, rb, rcv

    def tree_keyswitch(self, a, mask_size, per=1):
        return self.thr.mk_tree_keyswitch(a, self.planes, self._rows(per), mask_size)

    def ntt_mac(self, x, per=1):
        return self.thr.mk_ntt_mac(x, self.spectra, self._rows(per))
