"""The Python host layer's handle lifecycle on the CPU, against a recording stand-in for libzkb200.so: every handle is released
once whichever way it is closed, a child closed after its Context makes no library call, and Context.buffers() frees each
pointer once even when its block raises."""
import ctypes
import gc

import numpy as np
import pytest

import proof_systems_b200 as zk
from proof_systems_b200 import _lib


class RecordingLib:
    """Every zk_* call is logged and returns 0; an out-pointer (ctypes.byref of a c_void_p) receives a fresh nonzero handle, since a
    null c_void_p reads as false."""

    def __init__(self):
        self.calls, self._next = [], 0x1000

    def __getattr__(self, name):
        if not name.startswith("zk_"):
            raise AttributeError(name)

        def call(*args):
            self.calls.append((name, args))
            for a in args:
                out = getattr(a, "_obj", None)
                if isinstance(out, ctypes.c_void_p):
                    self._next += 0x100
                    out.value = self._next
            return 0
        return call

    def count(self, name):
        return sum(1 for n, _ in self.calls if n == name)

    def freed(self):
        """the pointers zk_dev_free received, in order"""
        return [args[1].value for n, args in self.calls if n == "zk_dev_free"]


@pytest.fixture
def fake(monkeypatch):
    rec = RecordingLib()
    monkeypatch.setattr(_lib, "_lib", rec)
    yield rec
    gc.collect()                  # whatever a test left open is released here, into the fake, before the real library is back


def fe(k=1):
    return np.ones((k, 4), dtype=np.uint64)


CHILDREN = {
    "Bases": (lambda ctx: zk.Bases(ctx, zk.PALLAS, np.ones((4, 8), dtype=np.uint64)), "zk_bases_free"),
    "SRS": (lambda ctx: zk.SRS(ctx, zk.PALLAS, np.ones((4, 8), dtype=np.uint64), np.ones(8, dtype=np.uint64)), "zk_srs_destroy"),
    "IndexCache": (lambda ctx: zk.IndexCache(ctx, b"MINAPK01"), "zk_index_cache_free"),
    "IndexCache.build": (lambda ctx: zk.IndexCache.build(ctx, zk.FP, zk.IndexHeader(), b"", b""), "zk_index_cache_free"),
    "IpaRounds": (lambda ctx: zk.IpaRounds(ctx, zk.Bases(ctx, zk.PALLAS, np.ones((2, 8), dtype=np.uint64)), fe(), fe()), "zk_ipa_free"),
    "LagrangeBasisEvaluations": (lambda ctx: zk.LagrangeBasisEvaluations(ctx, zk.FP, 16, 4, fe()), "zk_dev_free"),
}


def test_context_is_destroyed_once(fake):
    ctx = zk.Context(0)
    ctx.close()
    ctx.close()
    with zk.Context(0) as other:
        pass
    other.close()
    assert fake.count("zk_ctx_create") == 2 and fake.count("zk_ctx_destroy") == 2


@pytest.mark.parametrize("kind", sorted(CHILDREN))
def test_child_is_released_once(fake, kind):
    make, free = CHILDREN[kind]
    ctx = zk.Context(0)
    h = make(ctx)
    h.close()
    h.close()
    assert fake.count(free) == 1
    with make(ctx) as h2:
        assert fake.count(free) == 1
    h2.close()
    del h, h2
    gc.collect()
    assert fake.count(free) == 2
    ctx.close()


@pytest.mark.parametrize("kind", sorted(CHILDREN))
def test_child_closed_after_its_context_makes_no_call(fake, kind):
    make, free = CHILDREN[kind]
    ctx = zk.Context(0)
    h = make(ctx)
    ctx.close()
    n = len(fake.calls)
    h.close()
    del h
    gc.collect()
    assert len(fake.calls) == n and fake.count(free) == 0


def test_bases_free_is_close(fake):
    ctx = zk.Context(0)
    b = zk.Bases(ctx, zk.PALLAS, np.ones((4, 8), dtype=np.uint64))
    b.free()
    b.close()
    assert fake.count("zk_bases_free") == 1
    b = zk.Bases(ctx, zk.PALLAS, np.ones((4, 8), dtype=np.uint64))
    ctx.close()
    b.free()
    assert fake.count("zk_bases_free") == 1


def test_buffers_free_every_pointer_once_when_the_block_raises(fake):
    ctx = zk.Context(0)
    with pytest.raises(KeyError):
        with ctx.buffers() as bufs:
            ptrs = [bufs.put(fe(3)), bufs.alloc(64), bufs.put(np.zeros((0, 4), dtype=np.uint64))]
            raise KeyError("body")
    assert sorted(fake.freed()) == sorted(ptrs) and len(set(ptrs)) == 3 and all(ptrs)
    bufs.close()
    assert len(fake.freed()) == 3
    ctx.close()


def test_buffers_give_an_empty_array_32_bytes_and_upload_nothing(fake):
    with zk.Context(0) as ctx, ctx.buffers() as bufs:
        bufs.put(np.zeros((0, 4), dtype=np.uint64))
        sizes = [args[1] for n, args in fake.calls if n == "zk_dev_alloc"]
        assert sizes == [32] and fake.count("zk_dev_upload") == 0
        bufs.put(fe(2))
        assert [args[1] for n, args in fake.calls if n == "zk_dev_alloc"] == [32, 64] and fake.count("zk_dev_upload") == 1
    assert len(fake.freed()) == 2


def test_buffers_after_their_context_make_no_call(fake):
    ctx = zk.Context(0)
    bufs = ctx.buffers()
    bufs.alloc(32)
    ctx.close()
    bufs.close()
    assert fake.freed() == []
