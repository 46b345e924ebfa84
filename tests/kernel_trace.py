"""Which kernels a call ran, observed through torch.profiler (CUDA activity): the block-matching kernel families and their
template arguments, parsed from the demangled names the profiler reports (e.g.
`void vwb200::k1_fast_abs_kernel<3, false>(unsigned short const*, ...)`).  Used by the GPU tests through the `trace`
fixture, which a test module imports from here."""
import re

import numpy as np
import pytest

from bm_reference import expected_kernels

HOT = ("k1_fast_abs_kernel", "k1_screen_kernel", "k1_zone_int_kernel", "k1_generic_kernel")
MERGES = ("k1_fast_merge_kernel", "k1_screen_merge_kernel", "k1_generic_merge_kernel")
_KERNEL = re.compile(r"\b(k1_\w+?)(?:<([^>]*)>)?\(")
_printed = []


def _arg(a):
    """a template argument as an int: `3`, `(int)3`, `true`, `(bool)1`"""
    a = a.strip()
    if a in ("true", "false"):
        return int(a == "true")
    return int(re.findall(r"-?\d+", a)[-1])


def kernel_key(name):
    """(family, template arguments as ints) of a demangled kernel name, or None for kernels outside the k1 families"""
    m = _KERNEL.search(name)
    if not m:
        return None
    return m.group(1), tuple(_arg(a) for a in m.group(2).split(",")) if m.group(2) else ()


def inst_key(family, args):
    """(family, template arguments as ints): the form kernel_key() gives"""
    return family, tuple(int(a) for a in args)


class KernelTrace:
    """runs a callable under torch.profiler (CUDA activity) and keeps the names of the kernels it launched"""

    def run(self, fn):
        """fn() under the profiler.  A session loses the kernels launched right after it starts, so it opens with a warm-up
        step (a small torch kernel, not recorded) and records fn() in the step after it.  The call is deterministic: a
        session that still recorded no kernel of a hot family is traced again after a short pause, up to five times, and the
        test fails if none recorded one."""
        import time

        import torch
        from torch.profiler import ProfilerActivity, profile, schedule
        for attempt in range(5):
            if attempt:
                time.sleep(0.5)
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA], schedule=schedule(wait=0, warmup=1, active=1, repeat=1)) as prof:
                torch.ones(1, device="cuda").add_(1)
                torch.cuda.synchronize()
                prof.step()
                out = fn()
                torch.cuda.synchronize()
                prof.step()
            self.raw = [e.name for e in prof.events() if "vwb200" in e.name]
            self.keys = [k for k in map(kernel_key, self.raw) if k]
            if self.hot():
                break
        assert self.raw, "the profiler recorded no vwb200 kernel"
        assert self.hot(), f"the profiler recorded no block-matching kernel: {sorted(set(self.raw))}"
        if not _printed:
            _printed.append(True)
            print("kernel names as the profiler reports them:\n  " + "\n  ".join(sorted(set(self.raw))))
        return out

    def hot(self):
        return {k for k in self.keys if k[0] in HOT}

    def merges(self):
        return [k for k in self.keys if k[0] in MERGES]

    def assert_hot(self, cost, left, right, search, kernel, zone_int=False):
        """the hot kernel of the last run is the one the restated dispatch picks for these inputs"""
        (sx, sy), (kx, ky) = search, kernel
        l, r = np.asarray(left), np.asarray(right)
        vmin, vmax = float(min(l.min(), r.min())), float(max(l.max(), r.max()))
        integer = bool(np.all(l == np.rint(l)) and np.all(r == np.rint(r)))
        exp = expected_kernels(cost, l.shape[1] - kx + 1, l.shape[0] - ky + 1, sx, sy, kx, ky, vmin, vmax, integer, zone_int)
        want = {inst_key(exp.family, exp.args)} | ({inst_key("k1_fast_abs_kernel", exp.seed)} if exp.seed else set())
        assert self.hot() == want, f"ran {sorted(self.hot())}, expected {sorted(want)}"
        return exp


@pytest.fixture
def trace():
    """a KernelTrace; import it into a test module to use it there"""
    import torch
    torch.cuda.init()
    return KernelTrace()
