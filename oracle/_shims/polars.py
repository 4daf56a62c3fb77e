"""polars stand-in for the reference's dataset/utils.py (read_parquet + iter_rows(named=True) over pyarrow)."""
import pyarrow.parquet as _pq


class _Frame:
    def __init__(self, table):
        self._rows = table.to_pylist()

    def iter_rows(self, named=False):
        return iter(self._rows if named else [tuple(r.values()) for r in self._rows])


def read_parquet(path):
    return _Frame(_pq.read_table(path))
