"""A CPU test double for encrypted tables (DESIGN.md section 20).  TEST INFRASTRUCTURE ONLY.

The engine double of the multi-key machine on compressed keys (tests/multikey_pool_fake.py, which includes every other
multi-key, packing, compact and index double) plus the two indirect index levels of nufhe_b200.engine.Engine, composed
from the direct ones on the gathered tables: query q reads tables[table_ids[q]].  Every indirect call is recorded in
`indirect` as (kind, number of tables, table ids)."""
import numpy
import torch

from multikey_pool_fake import MultiKeyPoolFakeEngine


class EncryptedTableFakeEngine(MultiKeyPoolFakeEngine):

    def __init__(self):
        super().__init__()
        self.indirect = []

    def _gather(self, kind, tables, table_ids, queries):
        ids = numpy.asarray(table_ids, numpy.int64).reshape(-1)
        assert tables.dim() == 4 and ids.size == queries and 0 <= ids.min() and ids.max() < tables.shape[0]
        self.indirect.append((kind, tables.shape[0], ids.copy()))
        return tables[torch.from_numpy(ids)]

    def index_cmux_level_indirect(self, tables, table_ids, sel, bit, queries):
        return self.index_cmux_level(self._gather('cmux', tables, table_ids, queries), sel, bit, queries)

    def index_rotate_extract_indirect(self, tables, table_ids, sel, bits, columns, queries):
        return self.index_rotate_extract(self._gather('rotate', tables, table_ids, queries), sel, bits, columns, queries)
