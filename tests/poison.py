"""A pytest fixture that poisons every tensor torch.empty / torch.empty_like hands out: NaN for floating and complex
dtypes, all-ones bytes for integer dtypes, True for bool.  An output element or gradient a kernel forgets to write then
reads as NaN (or an impossible index) instead of whatever the caching allocator's recycled block held, which is often
the right value from the previous run.

The patch is on the torch module's attributes, not a TorchFunctionMode: a mode is thread-local, and CUDA backwards run on
autograd's device thread, where a mode set in the test would not apply.  The fixture counts calls per thread so that a
test can show that the backward's allocations went through it."""
import contextlib
import threading

import pytest
import torch


class Poison:
    def __init__(self):
        self.calls = 0
        self.threads = {}  # thread ident -> calls
        self._lock = threading.Lock()

    def wrap(self, fn):
        def poisoned(*args, **kwargs):
            t = fn(*args, **kwargs)
            with self._lock:
                self.calls += 1
                tid = threading.get_ident()
                self.threads[tid] = self.threads.get(tid, 0) + 1
            if t.numel() and t.device.type != "meta":
                with torch.no_grad():
                    if t.dtype.is_floating_point or t.dtype.is_complex:
                        t.fill_(float("nan"))
                    elif t.dtype == torch.bool:
                        t.fill_(True)
                    else:  # -1 for signed, the maximum for unsigned: every bit set
                        t.fill_(-1 if t.dtype.is_signed else torch.iinfo(t.dtype).max)
            return t
        return poisoned

    def off_thread_calls(self):
        """calls made on threads other than the caller's: the backward's allocations on autograd's device thread"""
        me = threading.get_ident()
        return sum(n for tid, n in self.threads.items() if tid != me)


@contextlib.contextmanager
def poisoning():
    p = Poison()
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(torch, "empty", p.wrap(torch.empty))
        mp.setattr(torch, "empty_like", p.wrap(torch.empty_like))
        yield p
        torch.cuda.synchronize()  # the backward's fills and kernels have run before the patch is lifted


@pytest.fixture
def poisoned():
    with poisoning() as p:
        yield p
