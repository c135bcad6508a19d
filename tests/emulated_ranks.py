"""K track-shard ranks emulated by K host threads of one process, meeting at a barrier for every all-reduce.

Each rank runs its own solve (the oracle's lm_solve or the CUDA lm_solve on its own stream and workspace; run_shards
gives each rank its shard of the tracks).  Every reduction goes through RankGroup.reduce: the rank stashes its operand,
passes the turn on and waits at a threading.Barrier whose action checks that all ranks arrived with the same (count, op)
tag, sums the operands in rank order (op 0) or takes their maximum (op 1, NaN-propagating) and hands the result back to
every rank.  A rank whose solve returns arrives once more with the tag "exit", so a rank that stops while the others ask
for another reduction breaks the barrier at once (RankGroup.error says how the tags differed) instead of waiting for the
timeout.

The turn is a lock that a rank holds whenever it runs anything but a barrier wait.  On the GPU this means that only one
rank has work in flight at a time and every wait happens on the host after a stream synchronisation: two solves never
overlap on the device, and a rank that fails ends in a host exception, not in a kernel waiting for another."""
import threading

import numpy as np

EXIT = "exit"


class RanksFailed(AssertionError):
    pass


class RankGroup:
    def __init__(self, K, timeout=120.0):
        self.K = K
        self.turn = threading.Lock()
        self.tags = [[] for _ in range(K)]          # every rank's sequence of reductions, "exit" last
        self.error = None
        self._arrived = [None] * K
        self._held = threading.local()
        self.barrier = threading.Barrier(K, action=self._combine, timeout=timeout)

    def _combine(self):
        tags = [a[0] for a in self._arrived]
        if any(t != tags[0] for t in tags):
            self.error = f"ranks diverged: arrived with {tags}"
            raise RanksFailed(self.error)
        if tags[0] == EXIT:
            return
        op = tags[0][1]
        vals = [a[1] for a in self._arrived]
        acc = vals[0].clone() if hasattr(vals[0], "clone") else vals[0].copy()
        for v in vals[1:]:
            if op == 0:
                acc += v
            elif hasattr(acc, "clone"):
                acc = acc.maximum(v)
            else:
                acc = np.maximum(acc, v)
        for a in self._arrived:
            a[2](acc)
        if hasattr(acc, "clone"):
            import torch
            torch.cuda.synchronize(acc.device)

    def _wait(self, rank, tag, value=None, writer=None):
        self.tags[rank].append(tag)
        self._arrived[rank] = (tag, value, writer)
        self._held.on = False
        self.turn.release()
        self.barrier.wait()

    def reduce(self, rank, count, op, value, writer):
        """all-reduce of `value` (numpy array or CUDA tensor of `count` doubles); writer(result) stores the result.
        Called holding the turn, returns holding it again."""
        try:
            self._wait(rank, (int(count), int(op)), value, writer)
        finally:
            self.turn.acquire()
            self._held.on = True

    def run(self, fn, join_timeout=600.0):
        """fn(rank) in K threads, each holding the turn; returns [fn(rank)].  Raises RanksFailed naming the ranks that
        failed (with RankGroup.error when the ranks diverged).  No thread outlives the call."""
        results, errors = [None] * self.K, [None] * self.K

        def body(rank):
            self.turn.acquire()
            self._held.on = True
            try:
                results[rank] = fn(rank)
                self._wait(rank, EXIT)
            except BaseException as e:              # noqa: BLE001 -- reported below, per rank
                errors[rank] = e
                self.barrier.abort()
            finally:
                if getattr(self._held, "on", False):
                    self._held.on = False
                    self.turn.release()

        threads = [threading.Thread(target=body, args=(r,), name=f"rank{r}", daemon=True) for r in range(self.K)]
        for t in threads:
            t.start()
        for t in threads:
            t.join(timeout=join_timeout)
        alive = [t.name for t in threads if t.is_alive()]
        if alive:
            self.barrier.abort()
            for t in threads:
                t.join(timeout=60.0)
            raise RanksFailed(f"ranks {alive} did not finish within {join_timeout} s")
        failed = {r: repr(e) for r, e in enumerate(errors) if e is not None}
        if failed:
            raise RanksFailed(f"{self.error or 'a rank failed'}; per rank: {failed}")
        for r in range(1, self.K):
            assert self.tags[r] == self.tags[0], ("reduction sequences differ", r, self.tags[r], self.tags[0])
        return results


def run_shards(N, K, body, device=None, timeout=120.0):
    """body(rank, lo, hi, hook) on K ranks, rank r on tracks shard_range(N, r, K) of N, with an OracleAllReduce hook,
    or with device a DeviceAllReduce hook and its own stream.  Returns ([body's result per rank], group); no rank
    thread is left alive."""
    from vggsfm_b200.dist import shard_range
    group = RankGroup(K, timeout=timeout)

    def rank(r):
        lo, hi = shard_range(N, r, K)
        if device is None:
            return body(r, lo, hi, OracleAllReduce(group, r))
        import torch
        st = torch.cuda.Stream(device=device)
        with torch.cuda.stream(st):
            out = body(r, lo, hi, DeviceAllReduce(group, r))
            st.synchronize()
        return out

    res = group.run(rank)
    assert not [t.name for t in threading.enumerate() if t.name.startswith("rank")]
    return res, group


class OracleAllReduce:
    """.sum / .max of oracle/ba_oracle.py lm_solve's `allreduce` argument over a RankGroup"""

    def __init__(self, group, rank):
        self.group, self.rank = group, rank

    def _reduce(self, a, op):
        out = {}
        self.group.reduce(self.rank, a.size, op, a.copy(), lambda acc: out.__setitem__("v", acc.copy()))
        return out["v"]

    def sum(self, arr):
        a = np.ascontiguousarray(arr, dtype=np.float64)
        return self._reduce(a.reshape(-1), 0).reshape(a.shape)

    def max(self, value):
        return float(self._reduce(np.array([float(value)]), 1)[0])


class DeviceAllReduce:
    """the `allreduce` argument of vggsfm_b200.bundle_adjustment.lm_solve over a RankGroup: like
    vggsfm_b200.dist.AllReduceHook, a view of the bound workspace is reduced in place"""

    fabric = None

    def __init__(self, group, rank):
        self.group, self.rank = group, rank
        self.calls = 0
        self._cb = None

    def bind(self, ws):
        import torch
        from vggsfm_b200 import _lib
        base = ws.data_ptr()

        def _fn(user, buf, count, op, stream):
            try:
                off = buf - base
                view = ws[off:off + count * 8].view(torch.float64)
                s = torch.cuda.ExternalStream(stream, device=ws.device)
                s.synchronize()
                with torch.cuda.stream(s):
                    stash = view.clone()
                s.synchronize()
                self.group.reduce(self.rank, count, op, stash, view.copy_)
                self.calls += 1
                return 0
            except Exception:                         # noqa: BLE001 -- rc != 0: lm_solve raises
                return -2

        self._cb = _lib.ALLREDUCE_FN(_fn)
        return self._cb
