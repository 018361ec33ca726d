"""One rank of the exact-integer tests of the multi-GPU block multiply (mb_matmul_blocked_dist and
mb_matmul_blocked_dist_host).  ctypes + numpy only: no torch.   argv: group rank world session [devices]

Runs the cases of one group of tests/dist_exact_cases.py on one communicator, in table order.  The operands of every
call are fresh integers from tests/exact_gemm.py whose products are exact in fp64 in any order and any split of K, so
each rank compares the C tiles it owns with `==` and, on a mismatch, fails with exact_gemm.report: the tile, how many
entries are wrong, where, and whether they are NaN (never written).  Each device call also reads mb_launch_count before
and after and fails unless the count names the path the case was built for."""
import ctypes as C
import os
import sys
import zlib
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import importlib.util                            # noqa: E402
# the ctypes declarations only — loaded by path, because importing the marlin_b200 PACKAGE would pull in torch
_spec = importlib.util.spec_from_file_location("mb_native_standalone", ROOT / "marlin_b200" / "_native.py")
nat = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(nat)
from tests import dist_exact_cases as cases     # noqa: E402
from tests import exact_gemm as xg              # noqa: E402

SENTINEL = -3.0e300                              # parent elements outside a C view must keep these bits
BF16_MAX = 256                                   # integers up to 2^8 are exact in bf16


def offsets(lens):
    return np.concatenate([[0], np.cumsum(lens)]).astype(int)


def make_operands(case, rep):
    """Full A (M x K), B (K x N) and the reference C for one call of `case`: the same on every rank."""
    rng = np.random.default_rng(zlib.crc32(f"{case.group}/{case.name}/{rep}".encode()))
    M, K, N = sum(case.rows), sum(case.ks), sum(case.cols)
    if getattr(case, "dtype", "f64") == "bf16":
        assert K * BF16_MAX * BF16_MAX < 2 ** 24, "fp32 accumulation must stay exact"
        A = rng.integers(-BF16_MAX, BF16_MAX + 1, size=(M, K)).astype(np.float64)
        B = rng.integers(-BF16_MAX, BF16_MAX + 1, size=(K, N)).astype(np.float64)
        s = rng.choice([-1.0, 1.0], size=K)
        A[0, :], B[:, 0] = BF16_MAX * s, BF16_MAX * s
        return A, B, A @ B
    A, B, _ = xg.operands(rng, M, K, N)
    ref = xg.reference(A, B)
    if getattr(case, "special", False):
        A, B, ref = add_special_values(case, A, B, ref)
    return A, B, ref


def add_special_values(case, A, B, ref):
    """One NaN in A row i0, one -Inf in A row i1 (both in the k segment of the rank that does not own C), one +Inf in a
    B column inside the owner's half, and zeros that meet the infinities (Inf * 0 = NaN).  The reference of every entry
    a special value reaches is classified from its element-wise products, as IEEE arithmetic defines them."""
    k0 = sum(case.ks[:case.grid[1] // 2])            # (1, k, 1), k even: rank 1 computes the upper half of K, rank 0 owns C
    i0, i1, iz, jc, jz = 3, 7, 11, 5, 9
    A, B = A.copy(), B.copy()
    A[i0, k0 + 1] = np.nan
    A[i1, k0 + 2] = -np.inf
    B[k0 + 3, jc] = np.inf
    B[k0 + 2, jz] = 0.0                              # (i1, jz): -Inf * 0
    A[iz, k0 + 3] = 0.0                              # (iz, jc): 0 * Inf
    fin_a, fin_b = np.where(np.isfinite(A), A, 0.0), np.where(np.isfinite(B), B, 0.0)
    ref = xg.reference(fin_a, fin_b)
    with np.errstate(invalid="ignore", over="ignore"):
        for i in range(A.shape[0]):
            for j in range(B.shape[1]):
                if i not in (i0, i1) and j != jc:
                    continue
                t = A[i, :] * B[:, j]
                if np.isnan(t).any() or (np.isposinf(t).any() and np.isneginf(t).any()):
                    ref[i, j] = np.nan
                elif np.isposinf(t).any():
                    ref[i, j] = np.inf
                elif np.isneginf(t).any():
                    ref[i, j] = -np.inf
                else:
                    ref[i, j] = fin_a[i, :] @ fin_b[:, j]
    assert np.isnan(ref[i1, jz]) and np.isnan(ref[iz, jc]) and np.isnan(ref[i0]).all()
    return A, B, ref


def same(got, want):
    """Equal as numbers, with NaN matching NaN and infinities matching in sign."""
    return np.array_equal(got, want, equal_nan=True)


class Rank:
    def __init__(self, rank, world, session, ndev):
        self.rank, self.world = rank, world
        self.lib = nat.load(build_if_missing=False)
        self.ctx = nat.c_ctx()
        nat.check(self.lib.mb_init(rank % ndev, C.byref(self.ctx)))
        self.comm = C.c_void_p()
        nat.check(self.lib.mb_comm_init(self.ctx, rank, world, session.encode(), C.byref(self.comm)))
        self.session = session
        self.handles = []                            # freed in reverse order: views before their parents
        self.failures = []                           # a mismatch is reported and the ranks go on in step

    def expect(self, ok, what):
        if not ok:
            self.failures.append(what)
            print(f"FAIL {what}", flush=True)
        return ok

    # ---------------------------------------------------------------------------------------------- device blocks
    def _keep(self, h):
        self.handles.append(h)
        return h

    def alloc(self, rows, cols, dtype=nat.MB_F64):
        h = nat.c_blk()
        nat.check(self.lib.mb_block_alloc(self.ctx, rows, cols, dtype, C.byref(h)))
        return self._keep(h)

    def upload(self, mat, layout="", dtype=nat.MB_F64):
        """A device block holding `mat` in one of the layouts of cases.VIEWS ("" = packed)."""
        f = np.asfortranarray(mat, dtype=np.float64)
        r, c = f.shape

        def packed(x):
            h = nat.c_blk()
            nat.check(self.lib.mb_block_upload(self.ctx, x.ctypes.data_as(C.c_void_p), 0, x.shape[0], x.shape[1], max(1, x.shape[0]), 0,
                                               dtype, C.byref(h)))
            return self._keep(h)

        if layout == "":
            return packed(f)
        if layout == "T":
            v = nat.c_blk()
            nat.check(self.lib.mb_block_view_t(self.ctx, packed(np.asfortranarray(f.T)), C.byref(v)))
            return self._keep(v)
        r0 = {"off16": 2, "off8": 1, "odd_ld": 0}[layout]
        pr = r + r0 + 2
        if (pr % 2 == 1) != (layout == "odd_ld"):
            pr += 1
        parent = self.alloc(pr, c)
        nat.check(self.lib.mb_block_fill(self.ctx, parent, SENTINEL))
        v = nat.c_blk()
        nat.check(self.lib.mb_block_slice(self.ctx, parent, r0, r0 + r, 0, c, C.byref(v)))
        self._keep(v)
        nat.check(self.lib.mb_block_copy(self.ctx, packed(f), v))
        return v

    def c_tile(self, rows, cols, view, dtype):
        """The owner's C tile, every element NaN: packed, or a slice of a SENTINEL-filled parent with an even leading
        dimension and a 16-byte aligned non-zero offset ("even") or with an odd leading dimension ("odd")."""
        if view == "":
            h = self.alloc(rows, cols, dtype)
            parent = None
        else:
            pr = rows + 4 + (rows % 2 if view == "even" else 1 - rows % 2)
            parent = self.alloc(pr, cols + 3)
            nat.check(self.lib.mb_block_fill(self.ctx, parent, SENTINEL))
            h = nat.c_blk()
            nat.check(self.lib.mb_block_slice(self.ctx, parent, 2, 2 + rows, 1, 1 + cols, C.byref(h)))
            self._keep(h)
        if dtype == nat.MB_F64:
            nat.check(self.lib.mb_block_fill(self.ctx, h, float("nan")))
        else:
            tmp = self.alloc(rows, cols)
            nat.check(self.lib.mb_block_fill(self.ctx, tmp, float("nan")))
            nat.check(self.lib.mb_block_copy(self.ctx, tmp, h))
        return h, parent

    def download(self, h, rows, cols):
        got = np.empty((rows, cols), order="F")
        nat.check(self.lib.mb_block_download(self.ctx, h, got.ctypes.data_as(C.c_void_p), max(1, rows)))
        return got

    def free_all(self):
        for h in reversed(self.handles):
            nat.check(self.lib.mb_block_free(self.ctx, h))
        self.handles = []

    # ---------------------------------------------------------------------------------------------- device entry
    def prepare(self, case, rep=0):
        """Operands and C tiles of one mb_matmul_blocked_dist call: everything but the call itself."""
        m, k, n = case.grid
        A, B, ref = make_operands(case, rep)
        ro, ko, co_ = offsets(case.rows), offsets(case.ks), offsets(case.cols)
        a_own, b_own = case.owners()
        dt = nat.MB_BF16 if case.dtype == "bf16" else nat.MB_F64
        a_view, b_view = dict(case.a_view), dict(case.b_view)
        a_h = (nat.c_blk * (m * k))()
        b_h = (nat.c_blk * (k * n))()
        c_h = (nat.c_blk * (m * n))()
        for t in range(m * k):
            if a_own[t] == self.rank:
                i, kk = divmod(t, k)
                a_h[t] = self.upload(A[ro[i]:ro[i + 1], ko[kk]:ko[kk + 1]], a_view.get(t, ""), dt)
        for t in range(k * n):
            if b_own[t] == self.rank:
                kk, j = divmod(t, n)
                b_h[t] = self.upload(B[ko[kk]:ko[kk + 1], co_[j]:co_[j + 1]], b_view.get(t, ""), dt)
        owner = (C.c_int32 * (m * n))()
        nat.check(self.lib.mb_dist_plan(m, k, n, self.world, None, owner))
        out_dt = nat.MB_F32 if case.dtype == "bf16" else nat.MB_F64
        mine = {}
        for t in range(m * n):
            if owner[t] == self.rank:
                i, j = divmod(t, n)
                h, parent = self.c_tile(case.rows[i], case.cols[j], case.c_view, out_dt)
                c_h[t] = h
                mine[t] = (h, parent, ref[ro[i]:ro[i + 1], co_[j]:co_[j + 1]])
        return dict(case=case, a_h=a_h, b_h=b_h, c_h=c_h, a_own=a_own, b_own=b_own, mine=mine, dtype=dt)

    def call(self, p):
        case = p["case"]
        m, k, n = case.grid
        os.environ["MARLIN_B200_DIST_SLOW"] = "1" if case.slow else "0"
        l0 = self.lib.mb_launch_count(self.ctx)
        nat.check(self.lib.mb_matmul_blocked_dist(self.comm, p["a_h"], (C.c_int32 * (m * k))(*p["a_own"]), p["b_h"],
                                                  (C.c_int32 * (k * n))(*p["b_own"]), m, k, n, (C.c_int32 * m)(*case.rows),
                                                  (C.c_int32 * k)(*case.ks), (C.c_int32 * n)(*case.cols), p["dtype"], p["c_h"]))
        launches = self.lib.mb_launch_count(self.ctx) - l0
        os.environ["MARLIN_B200_DIST_SLOW"] = "0"
        path = "fast" if launches <= case.fast_max else "general"
        self.expect(launches >= 1 and path == case.path,
                    f"{case.name}: rank {self.rank} made {launches} launches, the {path} path; the case is built for the {case.path} path")
        p["launches"], p["path"] = launches, path

    def check(self, p):
        case = p["case"]
        m, k, n = case.grid
        for t, (h, parent, want) in sorted(p["mine"].items()):
            i, j = divmod(t, n)
            got = self.download(h, case.rows[i], case.cols[j])
            if not self.expect(same(got, want), f"{case.name}: rank {self.rank}, C tile ({i}, {j}): {xg.report(got, want)}"):
                continue
            if parent is not None:
                pr = case.rows[i] + 4 + (case.rows[i] % 2 if case.c_view == "even" else 1 - case.rows[i] % 2)
                full = self.download(parent, pr, case.cols[j] + 3)
                outside = np.ones(full.shape, bool)
                outside[2:2 + case.rows[i], 1:1 + case.cols[j]] = False
                bits = full.view(np.uint64)[outside]
                bad = int(np.count_nonzero(bits != np.float64(SENTINEL).view(np.uint64)))
                self.expect(bad == 0, f"{case.name}: rank {self.rank}, C tile ({i}, {j}): {bad} parent elements outside the view changed")
        print(f"case {case.name}: rank {self.rank} launches {p['launches']} path {p['path']} exact ({len(p['mine'])} C tiles)",
              flush=True)

    def finish(self):
        nat.check(self.lib.mb_comm_check(self.comm))
        self.free_all()

    def device_case(self, case):
        p = self.prepare(case)
        self.call(p)
        self.check(p)
        self.finish()

    def queued(self, group):
        """Every call of `group` queued without a host synchronisation, then every result checked."""
        ps = [self.prepare(case) for case in group]
        nat.check(self.lib.mb_synchronize(self.ctx))
        nat.check(self.lib.mb_comm_barrier(self.comm))
        for p in ps:
            self.call(p)
        nat.check(self.lib.mb_synchronize(self.ctx))
        for p in ps:
            self.check(p)
        self.finish()

    # ---------------------------------------------------------------------------------------------- host entry
    def host_case(self, ci, case):
        lib, rank = self.lib, self.rank
        m, k, n = case.grid
        a_home = (C.c_int32 * (m * k))()
        b_home = (C.c_int32 * (k * n))()
        if case.a_home:
            a_home[:], b_home[:] = case.a_home, case.b_home
        else:
            nat.check(lib.mb_dist_host_homes(m, k, n, self.world, a_home, b_home))
        pr = (C.c_int32 * (m * k * n))()
        co = (C.c_int32 * (m * n))()
        nat.check(lib.mb_dist_plan(m, k, n, self.world, pr, co))
        rows, ks, cols = (C.c_int32 * m)(*case.rows), (C.c_int32 * k)(*case.ks), (C.c_int32 * n)(*case.cols)
        ro, ko, co_ = offsets(case.rows), offsets(case.ks), offsets(case.cols)
        held = sorted({s // k for s in range(m * k * n) if pr[s] == rank})        # C tiles I compute a partial of
        pc = (C.c_void_p * (m * n))()
        shared = {}
        if not case.error:
            for t in held:
                ptr = C.c_void_p()
                nbytes = case.rows[t // n] * case.cols[t % n] * 8
                nat.check(lib.mb_host_alloc_shared(f"{self.session}_{ci}_{t}".encode(), nbytes, C.byref(ptr)))
                shared[t] = (ptr, nbytes)
                pc[t] = ptr
        for rep in range(case.reps):
            A, B, ref = make_operands(case, rep)
            a_np = {t: np.asfortranarray(A[ro[t // k]:ro[t // k + 1], ko[t % k]:ko[t % k + 1]]) for t in range(m * k) if a_home[t] == rank}
            b_np = {t: np.asfortranarray(B[ko[t // n]:ko[t // n + 1], co_[t % n]:co_[t % n + 1]]) for t in range(k * n) if b_home[t] == rank}
            pa = (C.c_void_p * (m * k))(*[a_np[t].ctypes.data if t in a_np else None for t in range(m * k)])
            pb = (C.c_void_p * (k * n))(*[b_np[t].ctypes.data if t in b_np else None for t in range(k * n)])
            for t in shared:
                if co[t] == rank:
                    C.memset(shared[t][0], 0xFF, shared[t][1])           # NaN pattern: every byte must be overwritten
            nat.check(lib.mb_comm_barrier(self.comm))
            l0 = lib.mb_launch_count(self.ctx)
            rc = lib.mb_matmul_blocked_dist_host(self.comm, pa, a_home, pb, b_home, m, k, n, rows, ks, cols, pc)
            launches = lib.mb_launch_count(self.ctx) - l0
            if case.error:
                msg = lib.mb_last_error().decode("utf-8", "replace")
                self.expect(rc == nat.MB_ERR_UNSUPPORTED and case.error in msg, f"{case.name}: rank {rank} returned {rc}: {msg!r}")
                self.expect(launches == 0, f"{case.name}: rank {rank} launched {launches} kernels before refusing")
                print(f"host error {case.name}: {msg}", flush=True)
                break
            nat.check(rc)
            nat.check(lib.mb_comm_barrier(self.comm))                    # both holders have written their sub-blocks
            for t in held:
                if co[t] != rank:
                    continue
                i, j = divmod(t, n)
                got = np.ctypeslib.as_array(C.cast(shared[t][0], C.POINTER(C.c_double)), shape=(case.cols[j], case.rows[i])).T
                want = ref[ro[i]:ro[i + 1], co_[j]:co_[j + 1]]
                self.expect(same(got, want), f"{case.name}: rank {rank}, rep {rep}, C tile ({i}, {j}): {xg.report(got, want)}")
            nat.check(lib.mb_comm_barrier(self.comm))
            print(f"case {case.name}: rank {rank} rep {rep} launches {launches} exact", flush=True)
        for t in held:
            if t in shared:
                nat.check(lib.mb_host_free_shared(f"{self.session}_{ci}_{t}".encode(), shared[t][0], shared[t][1], 1 if co[t] == rank else 0))

    def close(self):
        nat.check(self.lib.mb_comm_barrier(self.comm))
        nat.check(self.lib.mb_comm_destroy(self.comm))
        nat.check(self.lib.mb_shutdown(self.ctx))


def main():
    group, rank, world, session = sys.argv[1], int(sys.argv[2]), int(sys.argv[3]), sys.argv[4]
    ndev = int(sys.argv[5]) if len(sys.argv) > 5 else world
    r = Rank(rank, world, session, ndev)
    todo = cases.group(group)
    for ci, case in enumerate(todo):
        assert case.world == world, f"{case.name} needs {case.world} ranks"
        if isinstance(case, cases.HostCase):
            r.host_case(ci, case)
        else:
            r.device_case(case)
    if group == "fresh":                            # the same communicator goes on with calls queued back to back
        r.queued(cases.group("queued"))
        todo = todo + cases.group("queued")
    r.close()
    assert "torch" not in sys.modules, "this worker must stay torch-free"
    if r.failures:
        sys.exit(f"exact rank {rank}/{world} FAILED group={group}: {len(r.failures)} mismatches\n" + "\n".join(r.failures))
    print(f"exact rank {rank}/{world} ok group={group} cases={len(todo)}", flush=True)


if __name__ == "__main__":
    main()
