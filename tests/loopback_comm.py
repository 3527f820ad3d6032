"""An in-process all-reduce(sum) over W ranks on one GPU, for the tests of the multi-rank PPO update (tests/test_gpu_ppo_multirank.py).

NCCL refuses two ranks on one device, and a test machine may have one GPU.  Here a rank is a host thread with its own CUDA stream, and
LoopbackGroup.fn is an ncclAllReduce-shaped ctypes callback (nn.ALL_REDUCE_FN) that uhc_ppo_trainer_set_all_reduce installs in a trainer; the
`comm` a rank passes is LoopbackGroup.comm(rank).  ctypes releases the GIL while a thread is inside the library, so the ranks run their updates
at once and meet inside the callback.

One call, on every rank:
  1. record `ready` on the rank's stream (after the producers of its buffer), post (count, buffer), meet the others at barrier 1;
  2. refuse a datatype other than float32, an op other than sum, or counts that differ between the ranks (NCCL would corrupt or hang);
  3. the stream waits on every rank's `ready` (all recorded before barrier 1), sums the ranks' buffers in rank order into a private buffer
     (so every rank gets the same bits) and records `read`;
  4. meet at barrier 2, the stream waits on every rank's `read` (the call is in place: another rank may still be reading this buffer), then
     copies the sum back.
A stream only ever waits on events recorded before a barrier its rank has passed, so no stream waits on work that is not enqueued, and every
barrier has a timeout: a rank that never arrives makes the others return non-zero instead of blocking.  Any exception in the callback returns
non-zero too (ctypes would otherwise report success for a callback that raised) and breaks the barriers so the other ranks stop waiting.
"""
import ctypes as C
import threading
import traceback

import torch

NCCL_FLOAT32, NCCL_SUM = 7, 0
ERR_REFUSED, ERR_BARRIER, ERR_COUNTS, ERR_EXCEPTION = 1, 2, 3, 4


class _DeviceArray:
    """n float32 at a device address, seen as a tensor through __cuda_array_interface__ (no copy, no ownership)"""

    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<f4", "data": (int(ptr), False), "strides": None, "version": 2}


def _view(ptr, n, device):
    return torch.as_tensor(_DeviceArray(ptr, n), device=device)


class LoopbackGroup:
    def __init__(self, world, device=0, timeout=60.0):
        from uhc_b200 import nn
        self.world, self.timeout = world, timeout
        self.device = torch.device("cuda", device)
        self._b1 = threading.Barrier(world, timeout=timeout)
        self._b2 = threading.Barrier(world, timeout=timeout)
        self._ready = [torch.cuda.Event() for _ in range(world)]
        self._read = [torch.cuda.Event() for _ in range(world)]
        self._posted = [None] * world
        self._priv = [None] * world
        self.log = [[] for _ in range(world)]       # per rank: (count, bytes) of every call that passed the argument checks
        self.errors = []                             # exceptions caught in the callback, as text
        self.fn = nn.ALL_REDUCE_FN(self._callback)

    @staticmethod
    def comm(rank):
        """the `comm` rank passes to uhc_ppo_update (non-NULL, as world > 1 requires)"""
        return C.c_void_p(rank + 1)

    def abort(self):
        """break both barriers: every rank waiting in (or later entering) a call returns non-zero at once"""
        self._b1.abort()
        self._b2.abort()

    def _callback(self, send, recv, count, datatype, op, comm, stream):
        try:
            return self.all_reduce((comm or 0) - 1, send, recv, count, datatype, op, stream)
        except BaseException:
            self.errors.append(traceback.format_exc())
            self.abort()
            return ERR_EXCEPTION

    def _private(self, rank, n, stream):
        buf = self._priv[rank]
        if buf is None or buf.numel() < n:
            with torch.cuda.stream(stream):      # the buffer is only ever used on this rank's stream: freeing it is stream-ordered
                buf = self._priv[rank] = torch.empty(n, device=self.device, dtype=torch.float32)
        return buf[:n]

    def all_reduce(self, rank, send, recv, count, datatype, op, stream):
        """the collective of one rank: send / recv device addresses, stream a cudaStream_t handle (int; 0 or None: the default stream)"""
        if datatype != NCCL_FLOAT32 or op != NCCL_SUM or not 0 <= rank < self.world or not send or not recv:
            self.errors.append(f"rank {rank}: refused datatype {datatype} op {op}")
            self.abort()
            return ERR_REFUSED
        st = torch.cuda.ExternalStream(stream, device=self.device) if stream else torch.cuda.default_stream(self.device)
        n = int(count)
        self._ready[rank].record(st)
        self._posted[rank] = (n, int(send))
        self.log[rank].append((n, 4 * n))
        try:
            self._b1.wait()
        except threading.BrokenBarrierError:
            return ERR_BARRIER
        posted = list(self._posted)             # read before barrier 2: no rank re-posts until every rank has passed it
        ok = len({c for c, _ in posted}) == 1
        if ok:
            acc = self._private(rank, n, st)
            with torch.cuda.stream(st):
                for e in self._ready:
                    st.wait_event(e)
                acc.copy_(_view(posted[0][1], n, self.device))
                for _, ptr in posted[1:]:
                    acc.add_(_view(ptr, n, self.device))
                self._read[rank].record(st)
        try:
            self._b2.wait()
        except threading.BrokenBarrierError:
            return ERR_BARRIER
        if not ok:
            self.errors.append(f"rank {rank}: the ranks' counts differ: {[c for c, _ in posted]}")
            return ERR_COUNTS
        with torch.cuda.stream(st):
            for e in self._read:
                st.wait_event(e)
            _view(recv, n, self.device).copy_(acc)
        return 0

    def run(self, fn, timeout=600.0):
        """fn(rank) on `world` threads, each with its own current stream on the group's device; returns [fn(rank)].  A rank that raises breaks
        the barriers (the others' collectives then fail fast) and its exception is re-raised here; every thread is joined."""
        results, errors = [None] * self.world, [None] * self.world

        def body(r):
            try:
                torch.cuda.set_device(self.device)
                s = torch.cuda.Stream(self.device)
                with torch.cuda.stream(s):
                    results[r] = fn(r)
                s.synchronize()
            except BaseException as e:
                errors[r] = (e, traceback.format_exc())
                self.abort()
        threads = [threading.Thread(target=body, args=(r,), daemon=True) for r in range(self.world)]
        for t in threads:
            t.start()
        for t in threads:
            t.join(timeout)
        alive = [r for r, t in enumerate(threads) if t.is_alive()]
        assert not alive, f"ranks {alive} did not finish within {timeout} s"
        for r, err in enumerate(errors):
            if err is not None:
                raise AssertionError(f"rank {r} failed:\n{err[1]}\ncollective errors: {self.errors}") from err[0]
        return results


class LoopbackGradComm:
    """nn.GradComm's interface (start / wait / pop_ms / bytes / calls) over a LoopbackGroup, for BatchedAgent.update_params' Python path"""

    def __init__(self, group, rank):
        self.group, self.rank, self.world = group, rank, group.world
        self.stream = torch.cuda.Stream(group.device)
        self.bytes, self.calls = 0, 0
        self.events = []

    def start(self, t):
        assert t.dtype == torch.float32 and t.is_contiguous()
        self.bytes += t.numel() * t.element_size(); self.calls += 1
        self.stream.wait_event(torch.cuda.current_stream().record_event())
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(self.stream)
        rc = self.group.all_reduce(self.rank, t.data_ptr(), t.data_ptr(), t.numel(), NCCL_FLOAT32, NCCL_SUM, self.stream.cuda_stream)
        if rc != 0:
            raise RuntimeError(f"loopback all-reduce failed with code {rc}: {self.group.errors}")
        e1.record(self.stream)
        self.events.append((e0, e1))
        return e1

    def wait(self, done=None):
        if done is not None:
            torch.cuda.current_stream().wait_event(done)
        else:
            torch.cuda.current_stream().wait_stream(self.stream)

    def pop_ms(self):
        ms = sum(a.elapsed_time(b) for a, b in self.events)
        self.events = []
        return ms
