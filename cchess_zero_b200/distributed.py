"""The one collective of the path: all_gather of finished-game (s, pi, z) tuples (SURVEY 8(e)).

Games are independent, so ranks never communicate during search; when games end, each rank packs its new tuples into
fixed-size records and one all_gather_into_tensor (NCCL over NVLink on GPUs, gloo in the CPU tests) gives every rank
the whole batch for its replay buffer (main.py:1234-1240 feeds data_buffer).

Off the critical path (VERDICT r1 item 8): packing is vectorised per game, the gathered buffer is sized to the largest
rank's count of THIS round (a 4-byte-per-rank count gather first: nothing is dropped, nothing fixed-size is shipped), the
payload gather is launched with async_op=True and its device->host copy lands in pinned memory on a side stream while the
next ply's search runs; `finish()` is called one step later and unpacks lazily (arrays first, python tuples on request)."""
import numpy as np
import torch
import torch.distributed as dist

MAXC = 128
# record = canonical (side-to-move) board 90 B | side 1 | n 1 | pad 4 | int16 label[128] | f64 prob[128] | f64 z
O_SIDE, O_N, O_IDX, O_PROB, O_Z = 90, 91, 96, 96 + 2 * MAXC, 96 + 2 * MAXC + 8 * MAXC
REC_BYTES = O_Z + 8


def pack_records(records, cap=None):
    """records: iterable of GameRecord (selfplay.py).  Returns (uint8 [n, REC_BYTES], n, leftover records): with cap=None
    every tuple is packed; with a cap whole trailing games that do not fit are handed back, never dropped."""
    rows, n, left = [], 0, []
    records = list(records)
    for k, r in enumerate(records):
        L = len(r)
        if cap is not None and n + L > cap:
            left = records[k:]
            break
        if L == 0:
            continue
        p = r.positions()
        buf = np.zeros((L, REC_BYTES), dtype=np.uint8)
        buf[:, :90] = p.boards
        buf[:, O_SIDE] = p.sides
        buf[:, O_N] = p.n
        buf[:, O_IDX:O_PROB] = p.idx.view(np.uint8)
        buf[:, O_PROB:O_Z] = p.prob.view(np.uint8)
        buf[:, O_Z:] = p.z.reshape(L, 1).view(np.uint8)
        rows.append(buf)
        n += L
    out = np.concatenate(rows) if rows else np.zeros((0, REC_BYTES), dtype=np.uint8)
    return out, n, left


class TupleBatch:
    """Gathered tuples as arrays; python tuples (state str, pi dense float64 [2086], z) only on request."""

    def __init__(self, buf):
        buf = np.ascontiguousarray(buf, dtype=np.uint8).reshape(-1, REC_BYTES)
        self.boards = buf[:, :90].copy()                                           # side-to-move canonical boards
        self.n = buf[:, O_N].astype(np.int64)
        self.idx = np.ascontiguousarray(buf[:, O_IDX:O_PROB]).view(np.int16).reshape(-1, MAXC)
        self.prob = np.ascontiguousarray(buf[:, O_PROB:O_Z]).view(np.float64).reshape(-1, MAXC)
        self.z = np.ascontiguousarray(buf[:, O_Z:]).view(np.float64).reshape(-1)

    def __len__(self):
        return self.boards.shape[0]

    def dense_pi(self):
        pi = np.zeros((len(self), 2086))
        valid = np.arange(MAXC)[None, :] < self.n[:, None]
        r = np.nonzero(valid)[0]
        pi[r, self.idx[valid].astype(np.int64)] = self.prob[valid]
        return pi

    def tuples(self):
        from . import rules
        pi = self.dense_pi()
        return [(rules.board_to_state(b), pi[i], float(self.z[i])) for i, b in enumerate(self.boards)]


def unpack_records(buf, n):
    """-> list of (state str, pi dense float64 [2086], z float)"""
    return TupleBatch(np.asarray(buf)[:n]).tuples()


class AsyncTupleGather:
    """Pipelined gather with no host synchronisation on the step's critical path:
         start(records) at step s      packs this rank's finished games and launches an ASYNC all_gather of the per-rank counts;
         start(...) at step s + 1       reads the (long finished) counts of step s, sizes the payload exactly and launches its async
                                        all_gather + device->host copy on a side stream;
         finish()                       returns the TupleBatch of every payload that has landed (usually the one of step s - 1).
       drain() completes everything in flight (end of a run).  Nothing is dropped and nothing fixed-size is shipped."""

    def __init__(self, device, group=None):
        self.device, self.group = torch.device(device), group
        self.world = dist.get_world_size(group)
        self.cuda = self.device.type == "cuda"
        self.side = torch.cuda.Stream(self.device) if self.cuda else None
        self._counting = []      # stage 1: (buf, k, count tensor, all-counts tensor, work)
        self._moving = []        # stage 2: (counts, m, allr / host, event or work)
        self.bytes_gathered = 0

    def _launch_payload(self):
        while self._counting:
            buf, k, cnt, allc, work = self._counting.pop(0)
            work.wait()
            counts = allc.cpu().numpy().astype(np.int64)
            m = int(counts.max())
            if m == 0:
                self._moving.append((counts, 0, None, None))
                continue
            mine = torch.zeros((m, REC_BYTES), dtype=torch.uint8, device=self.device)
            if k:
                src = torch.from_numpy(buf)
                mine[:k].copy_(src.pin_memory() if self.cuda else src, non_blocking=True)
            allr = torch.empty((self.world * m, REC_BYTES), dtype=torch.uint8, device=self.device)
            w2 = dist.all_gather_into_tensor(allr, mine, group=self.group, async_op=True)
            if self.cuda:
                host = torch.empty((self.world * m, REC_BYTES), dtype=torch.uint8).pin_memory()
                with torch.cuda.stream(self.side):
                    w2.wait()                                                      # the side stream waits for the collective only
                    host.copy_(allr, non_blocking=True)
                    ev = torch.cuda.Event()
                    ev.record(self.side)
                self._moving.append((counts, m, (allr, mine, host), ev))
            else:
                self._moving.append((counts, m, allr, w2))
            self.bytes_gathered += int(self.world * m * REC_BYTES)

    def start(self, records):
        self._launch_payload()                                                     # counts of the previous step(s) are in by now
        buf, k, _ = pack_records(records)
        cnt = torch.tensor([k], dtype=torch.int32, device=self.device)
        allc = torch.empty((self.world,), dtype=torch.int32, device=self.device)
        work = dist.all_gather_into_tensor(allc, cnt, group=self.group, async_op=True)    # 4 B per rank; nobody waits for it here
        self._counting.append((buf, k, cnt, allc, work))

    def _take(self, block):
        out = []
        while self._moving:
            counts, m, data, sync = self._moving[0]
            if m and self.cuda and not block and not sync.query():
                break
            self._moving.pop(0)
            if m == 0:
                continue
            if self.cuda:
                sync.synchronize()
                arr = data[2].numpy()
            else:
                sync.wait()
                arr = data.numpy()
            arr = arr.reshape(self.world, m, REC_BYTES)
            out.extend(arr[r, :int(counts[r])] for r in range(self.world))
        return out

    def finish(self, block=False):
        """TupleBatch of every rank's tuples whose payload has landed (rank-major per round); None when nothing is ready."""
        parts = self._take(block)
        return TupleBatch(np.concatenate(parts)) if parts else None

    def drain(self):
        """Complete every round in flight (collective: every rank must call it)."""
        self._launch_payload()
        parts = self._take(True)
        return TupleBatch(np.concatenate(parts)) if parts else TupleBatch(np.zeros((0, REC_BYTES), dtype=np.uint8))


def all_gather_tuples(records, device, cap=None, group=None):
    """Synchronous convenience form: every rank contributes ALL its tuples (`cap` is accepted for compatibility and ignored:
    the payload is sized from the gathered counts); returns the list of all ranks' tuples (rank-major)."""
    g = AsyncTupleGather(device, group)
    g.start(records)
    return g.drain().tuples()


def shard_seeds(n_games_per_rank, rank, base_seed=0):
    """Per-game RNG seeds that do not depend on the world size: game g of rank r gets base + r*n + g."""
    return [base_seed + rank * n_games_per_rank + g for g in range(n_games_per_rank)]
