"""The evaluation tail's summation order restated on the host, and the ctypes driver of tests/exchange_harness.cu.

Order (optim_kernels.cuh: reduce_block_entries, combine8, exchange_block): on each rank, warp w of a tail block adds the per-CTA
partials of CTAs b = w, w + 8, ... in increasing b, starting from 0.0; the eight warp sums are combined as
((0+1)+(2+3))+((4+5)+(6+7)) (combine8).  The exchange then puts rank k's local sum in slot k of eight, ranks >= world
contributing 0.0, and combines the slots with combine8 again.  numpy's float64 additions round exactly as the device's, so the
restatement is the kernels' result bit for bit.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np

TESTS = os.path.dirname(os.path.abspath(__file__))
PKG = os.path.join(os.path.dirname(TESTS), "pinns-tf2.0_b200")
# PINN_CSRC: the kernel sources of another build of the library (PINN_LIB), e.g. a mutant of tests/kernel_mutants.py
CSRC = os.environ.get("PINN_CSRC") or os.path.join(PKG, "csrc")
SOURCE = os.path.join(TESTS, "exchange_harness.cu")
P2P_MAX = 8
RING = 16                        # loss ring entries of the harness


def combine8(v):
    return ((v[0] + v[1]) + (v[2] + v[3])) + ((v[4] + v[5]) + (v[6] + v[7]))


def columns(p_net, extra_src):
    """Source column of every entry of R (pinn::ReduceMap)."""
    return np.concatenate([np.arange(p_net), np.asarray(extra_src, dtype=np.int64)]).astype(np.int64)


def local_sum(partials, cols):
    """One rank's reduction of its per-CTA partials (n_cta x stride) into the entries `cols`."""
    p = np.asarray(partials, dtype=np.float64)[:, cols]
    acc = np.zeros((8, p.shape[1]))
    for b in range(p.shape[0]):
        acc[b % 8] = acc[b % 8] + p[b]
    return combine8(acc)


def exchanged(local_sums):
    """The rank-ordered sum every rank computes from the ranks' local sums."""
    if not 1 <= len(local_sums) <= P2P_MAX:
        raise ValueError("1..8 ranks")
    slots = np.zeros((P2P_MAX, len(local_sums[0])))
    slots[:len(local_sums)] = local_sums
    return combine8(slots)


def tail_sum(partials_per_rank, cols):
    return exchanged([local_sum(p, cols) for p in partials_per_rank])


def cancelling(rng, n_cta, stride):
    """Partials whose sums cancel heavily: magnitudes spread over 2^-30 .. 2^30 with random signs, and every CTA's large
    values undone by a later CTA's, so that any other order of the additions changes the low bits."""
    mant = rng.uniform(1.0, 2.0, (n_cta, stride)) * rng.choice([-1.0, 1.0], (n_cta, stride))
    x = np.ldexp(mant, rng.integers(-30, 31, (n_cta, stride)))
    if n_cta > 1:
        big = np.ldexp(rng.uniform(1.0, 2.0, stride), 40)
        x[0] += big
        x[-1] -= big * (1.0 + 2.0 ** -40)
    return x


def cancelling_ranks(rng, n_ctas, stride):
    """cancelling() partials for each rank, with a further large value added on rank 0 and taken back on rank 1: the
    exchange adds those two first, and any other pairing of the ranks rounds the others' sums at the large value's scale."""
    parts = [cancelling(rng, n, stride) for n in n_ctas]
    if len(parts) > 1:
        big = np.ldexp(rng.uniform(1.0, 2.0, stride), 50)
        parts[0][0] += big
        parts[1][-1] -= big * (1.0 - 2.0 ** -20)
    return parts


# ---------------------------------------------------------------------------------------------------------------- the harness
def compile_harness(out_dir):
    """exchange_harness.cu with the library's nvcc flags (pinns-tf2.0_b200/build.py) into out_dir; returns the .so path."""
    if PKG not in sys.path:
        sys.path.insert(0, PKG)
    import build as pinn_build
    out = os.path.join(out_dir, "exchange_harness.so")
    cmd = [pinn_build._nvcc()] + pinn_build.NVCC_FLAGS + ["-I", CSRC, "-o", out, SOURCE, "-lcudart"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + " ".join(cmd) + "\n" + r.stdout + r.stderr)
    return out


_dp, _ip = C.POINTER(C.c_double), C.POINTER(C.c_int)


def _d(a):
    return a.ctypes.data_as(_dp)


class Harness(object):
    """W simulated ranks: per rank and evaluation slot a partial vector; enqueue() runs one evaluation on every rank (form
    "reduce": pinn::reduce_tail; "fused": pinn::fused_tail in a launch of n_cta CTAs; "adam_update": pinn::adam_update on R) and
    snapshots every rank's state; read() returns a snapshot after sync()."""
    FORMS = {"reduce": 0, "fused": 1, "adam_update": 2}

    def __init__(self, lib_path, world, p_net, extra_src, stride, max_cta=1, n_slots=1, n_snap=1):
        lib = C.CDLL(lib_path)
        lib.xh_create.restype = C.c_void_p
        lib.xh_create.argtypes = [C.c_int] * 4 + [_ip] + [C.c_int] * 4
        for name, args in (("xh_info", [C.c_void_p, _ip]), ("xh_load", [C.c_void_p, C.c_int, C.c_int, _dp, C.c_int, C.c_int]),
                           ("xh_set_state", [C.c_void_p, C.c_int, _dp, _dp, _dp, C.c_int]),
                           ("xh_enqueue", [C.c_void_p, C.c_int, C.c_int, _ip, C.c_int, _dp, C.c_int]),
                           ("xh_sync", [C.c_void_p]), ("xh_read", [C.c_void_p, C.c_int, C.c_int, _dp, _ip]),
                           ("xh_read_flags", [C.c_void_p, C.c_int, C.POINTER(C.c_ulonglong)]),
                           ("xh_destroy", [C.c_void_p]), ("xh_last_cuda_error", [])):
            getattr(lib, name).restype = C.c_int
            getattr(lib, name).argtypes = args
        self.lib, self.world, self.stride = lib, world, stride
        self.cols = columns(p_net, extra_src)
        self.n_out = len(self.cols)
        self.P = self.n_out - 3
        ex = (C.c_int * 8)(*list(extra_src))
        self.h = lib.xh_create(world, self.n_out, p_net, len(extra_src), ex, stride, max_cta, n_slots, n_snap)
        if not self.h:
            raise RuntimeError("xh_create failed (CUDA error %d)" % lib.xh_last_cuda_error())
        info = (C.c_int * 3)()
        lib.xh_info(self.h, info)
        self.sms, self.occ_reduce, self.occ_fused = info[0], info[1], info[2]
        self.nb = (self.n_out + 31) // 32
        self.slot_len, self.n_blocks = (self.n_out + 15) // 16 * 16, self.nb

    def _ck(self, rc, what):
        if rc != 0:
            raise RuntimeError("%s failed (rc %d, CUDA error %d)" % (what, rc, self.lib.xh_last_cuda_error()))

    def reduce_grid(self):
        """launch_tail's grid (nb, capped at 2 x SMs), shrunk so that the grids of all ranks are resident at once."""
        return min(self.nb, 2 * self.sms, self.occ_reduce * self.sms // self.world)

    def load(self, rank, slot, partials, run_flag=0):
        p = np.ascontiguousarray(partials, dtype=np.float64)
        assert p.ndim == 2 and p.shape[1] == self.stride
        self._ck(self.lib.xh_load(self.h, rank, slot, _d(p), p.shape[0], int(run_flag)), "xh_load")

    def set_state(self, rank, w, m, v, step0):
        w, m, v = (np.ascontiguousarray(a, dtype=np.float64) for a in (w, m, v))
        assert w.size == m.size == v.size == self.P
        self._ck(self.lib.xh_set_state(self.h, rank, _d(w), _d(m), _d(v), int(step0)), "xh_set_state")

    def enqueue(self, slot, form, adam=None, snap=0, grid=None):
        g = grid if grid is not None else [self.reduce_grid()] * self.world
        gr = (C.c_int * self.world)(*g)
        hp = np.array(adam if adam is not None else (0.0, 0.0, 0.0, 0.0), dtype=np.float64)
        rc = self.lib.xh_enqueue(self.h, slot, self.FORMS[form], gr, 1 if adam is not None else 0, _d(hp), snap)
        if rc == -2:
            raise RuntimeError("the ranks' grids cannot all be resident at once")
        self._ck(rc, "xh_enqueue")

    def sync(self):
        self._ck(self.lib.xh_sync(self.h), "xh_sync")

    def read(self, rank, snap=0):
        n, P = self.n_out, self.P
        out = np.empty(n + 3 * P + RING)
        ints = (C.c_int * 5)()
        self._ck(self.lib.xh_read(self.h, rank, snap, _d(out), ints), "xh_read")
        return dict(R=out[:n], w=out[n:n + P], m=out[n + P:n + 2 * P], v=out[n + 2 * P:n + 3 * P], ring=out[n + 3 * P:],
                    step=list(ints[:3]), xseq=ints[3], err=ints[4])

    def flags(self, rank):
        """The exchange flags of `rank`'s buffer as they stand: [2 parities][world][n_blocks]."""
        out = (C.c_ulonglong * (2 * self.world * self.n_blocks))()
        self._ck(self.lib.xh_read_flags(self.h, rank, out), "xh_read_flags")
        return np.array(out[:], dtype=np.uint64).reshape(2, self.world, self.n_blocks)

    def close(self):
        if self.h:
            self.lib.xh_destroy(self.h)
            self.h = None
