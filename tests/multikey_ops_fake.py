"""A CPU test double for the multi-key tree LUTs, packing, expansion and index lookups (DESIGN.md section 18).  TEST
INFRASTRUCTURE ONLY.

The multi-key engine double (tests/multikey_fake.py) joined with the tree, packing and compact doubles of the CPU suite,
the encrypted-index steps composed from tests/index_ref.py, and the three new multi-key calls composed per tenant from
the single-key ones, so that nufhe_b200/multikey.py runs in the CPU suite against exactly what per-tenant
VirtualMachines compute."""
import numpy
import torch

from fake_engine import N, _np, _t
from multikey_fake import MultiKeyFakeEngine
from test_host_compact import CompactFakeEngine
from test_host_tree_lut import TreeFakeEngine
import index_ref


class MultiKeyOpsFakeEngine(MultiKeyFakeEngine, TreeFakeEngine, CompactFakeEngine):

    # --- encrypted-index steps: selector "spectra" are the reference's transformed rows
    def index_prepare(self, ggsw):
        rows = ggsw.numel() // (8 * N)
        return _t(index_ref.transform(_np(ggsw))).reshape(rows, -1)

    @staticmethod
    def _sel(sel, queries):
        return _np(sel, True).reshape(-1, 2, 2, 2, N), sel.shape[1]

    @staticmethod
    def _nodes(x, queries):
        x = _np(x)
        return numpy.ascontiguousarray(numpy.broadcast_to(x, (queries,) + x.shape[-3:]) if x.ndim == 3 else x)

    def index_cmux_level(self, x, sel, bit, queries):
        sel_ref, m = self._sel(sel, queries)
        return _t(index_ref.cmux_level(self._nodes(x, queries), sel_ref, numpy.arange(queries) * m + bit))

    def index_rotate_extract(self, acc, sel, bits, columns, queries):
        sel_ref, m = self._sel(sel, queries)
        rows = numpy.arange(queries)[:, None] * m + numpy.arange(m)[None, :]
        a, b = index_ref.rotate_extract(self._nodes(acc, queries), sel_ref, rows, bits, columns)
        return _t(a), _t(b)

    # --- the multi-key calls of section 18, composed per tenant
    def mk_bootstrap_lut_extract(self, x1, x2, c, s1, s2, tv, log2_outputs, bk_ints, counts):
        if tv.dim() == 1:
            return super().mk_bootstrap_lut_extract(x1, x2, c, s1, s2, tv, log2_outputs, bk_ints, counts)
        assert len(bk_ints) == len(counts) and sum(counts) == x1[1].numel() == tv.shape[0]
        return self._cat([self.bootstrap_lut_extract(self._rows(x1, lo, hi), self._rows(x2, lo, hi), c, s1, s2,
                                                     tv[lo:hi], log2_outputs, bk_ints[t])
                          for t, lo, hi in self._segments(counts) if hi > lo], N)

    def mk_bootstrap_glwe_lut_extract(self, x, tv, bk_ints, counts):
        assert len(bk_ints) == len(counts) and sum(counts) == x[1].numel()
        return self._cat([self.bootstrap_glwe_lut_extract(self._rows(x, lo, hi), tv[lo:hi], bk_ints[t])
                          for t, lo, hi in self._segments(counts) if hi > lo], N)

    def mk_tree_keyswitch(self, a, planes, counts, mask_size):
        assert len(planes) == len(counts) and sum(counts) == a.shape[0]
        parts = [self.tree_keyswitch(a[lo:hi], planes[t], mask_size) for t, lo, hi in self._segments(counts) if hi > lo]
        return torch.cat(parts) if parts else torch.empty((0, mask_size + 1, N), dtype=torch.int32)

    def mk_ntt_mac(self, x, keys, group_counts):
        assert len(keys) == len(group_counts) and sum(group_counts) == x.shape[0]
        parts = [self.ntt_mac(x[lo:hi], keys[t]) for t, lo, hi in self._segments(group_counts) if hi > lo]
        return torch.cat(parts)
