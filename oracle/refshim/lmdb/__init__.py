"""Read-only stand-in for the `lmdb` package, for oracle/pin_dataset.py only: ``open(path).begin().get(key)`` reads the
one-file-per-key directory store of lav_b200.data_paint.DirEnv, so the reference's BasicDataset runs on a synthetic recording."""
import builtins
import os


class _Txn:
    def __init__(self, path):
        self.path = path

    def get(self, key):
        fn = os.path.join(self.path, "kv", key.decode() if isinstance(key, bytes) else key)
        if not os.path.exists(fn):
            return None
        with builtins.open(fn, "rb") as f:
            return f.read()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        return False


class _Env:
    def __init__(self, path):
        self.path = path

    def begin(self, write=False):
        assert not write, "the stand-in is read-only"
        return _Txn(self.path)


def open(path, **kwargs):        # noqa: A001 (the lmdb API's name)
    return _Env(path)
