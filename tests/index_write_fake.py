"""A CPU test double for oblivious writes (DESIGN.md section 21).  TEST INFRASTRUCTURE ONLY.

The encrypted-table engine double (tests/encrypted_table_fake.py) plus the three write calls of
nufhe_b200.engine.Engine composed from tests/write_ref.py; the last level adds into the accumulators in place."""
import numpy
import torch

from fake_engine import _np, _t
from encrypted_table_fake import EncryptedTableFakeEngine
import write_ref


class IndexWriteFakeEngine(EncryptedTableFakeEngine):

    def index_write_assemble(self, v, b, bits):
        return _t(write_ref.assemble(None if v is None else _np(v), _np(b), bits))

    def _add(self, acc, leaves, table_ids):
        ids = numpy.zeros(leaves.shape[0], numpy.int64) if table_ids is None else numpy.asarray(table_ids, numpy.int64)
        acc.copy_(_t(write_ref.accumulate(_np(acc), leaves, ids)))

    def index_write_rotate(self, delta, sel, bits, acc=None, table_ids=None):
        Q = delta.shape[0]
        sel_ref, m = self._sel(sel, Q)
        rows = numpy.arange(Q)[:, None] * m + numpy.arange(min(bits, 10))[None, :]
        out = write_ref.rotate(_np(delta), sel_ref, rows)
        assert (acc is None) == (bits > 10)
        if acc is None:
            return _t(out)
        self._add(acc, out, table_ids)

    def index_demux_level(self, x, sel, bit, acc=None, table_ids=None):
        Q = x.shape[0]
        sel_ref, m = self._sel(sel, Q)
        out = write_ref.demux_level(_np(x), sel_ref, numpy.arange(Q) * m + bit)
        if acc is None:
            return _t(out)
        self._add(acc, out, table_ids)
