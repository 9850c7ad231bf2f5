"""The training loop on one GPU: self-play -> device replay buffer -> policy_update -> arena gate -> promotion.

The reference trains with run() (main.py:1224-1248): one game of self-play, its tuples through state_to_positions into a
deque(maxlen=buffer_size), and one policy_update (main.py:1157-1205) per game once the deque holds more than batch_size tuples.
Here thousands of games play at once (SelfPlay), finished games go into a ring of device arrays in the compact record format
of distributed.pack_records (canonical board, sparse pi, z), and one kernel (cz_replay_batch) turns sampled ring rows into
the f32 planes / dense pi / z mini-batch that train_step_module consumes.  No tuple ever becomes a Python string or a dense
host array.

    ReplayBuffer   the ring: add(TupleBatch), sample_rows(rng, k) (= random.sample over the deque), batch(rows, mirror)
    Trainer        the loop; policy_update() keeps the reference's update rule, KL early stop and lr_multiplier adaptation
    policy_kl / next_lr_multiplier / explained_variance
                   the arithmetic after the forward passes, shared with cchess_main.policy_update
    main()         python -m cchess_zero_b200.train ...: one JSON line per report interval"""
import argparse
import contextlib
import ctypes as C
import json
import math
import os
import random
import sys
import tempfile
import time
import types

import numpy as np
import torch

from ._lib import MAXCHILD, NLABEL, NSQ, check, lib
from .distributed import TupleBatch, pack_records


# ---- the arithmetic of policy_update after its forward passes (main.py:1176-1201) --------------------------------------
def policy_kl(old_probs, new_probs):
    """mean over rows of sum(old * log((old + 1e-10) / (new + 1e-10))).  main.py:1178-1182 drops the terms whose str() is 'nan' or
    'inf' -- and therefore KEEPS '-inf' (logits are used as probabilities, so negative old_probs are routine and a row sum can
    legitimately be -inf)."""
    with np.errstate(all="ignore"):
        kl_tmp = old_probs * (np.log((old_probs + 1e-10) / (new_probs + 1e-10)))
    return np.mean([np.sum(line[~(np.isnan(line) | np.isposinf(line))]) for line in kl_tmp])


def next_lr_multiplier(kl, kl_targ, lr_multiplier):
    """main.py:1190-1193: divide by 1.5 above 2 kl_targ (down to 0.1), multiply by 1.5 below kl_targ / 2 (up to 10)."""
    if kl > kl_targ * 2 and lr_multiplier > 0.1:
        lr_multiplier /= 1.5
    elif kl < kl_targ / 2 and lr_multiplier < 10:
        lr_multiplier *= 1.5
    return lr_multiplier


def explained_variance(winner_batch, v):
    """main.py:1194-1197: 1 - var(z - v) / var(z), z the [B,1] winner batch and v flattened -- the reference's expression as written
    (the subtraction broadcasts to [B,B])."""
    wb = np.array(winner_batch)
    return 1 - np.var(wb - np.asarray(v).flatten()) / np.var(wb)


# ---- records -------------------------------------------------------------------------------------------------------------
_MIRROR = None


def mirror_labels():
    """int16 [2086]: the label of each label's left-right mirrored move (file x -> 8 - x), cz_mirror_labels.  The library checks
    that the table is closed under the mirror and an involution and refuses to hand it out otherwise."""
    global _MIRROR
    if _MIRROR is None:
        m = np.zeros(NLABEL, dtype=np.int16)
        check(lib().cz_mirror_labels(m.ctypes.data_as(C.c_void_p)), "cz_mirror_labels")
        _MIRROR = m
    return _MIRROR


def validate_tuples(tb):
    """Checks records before they enter the replay buffer (anything with boards [L,90], n [L], idx [L,128], prob [L,128], z [L]
    arrays, e.g. a TupleBatch); raises ValueError.  Piece codes 0..14, 0 <= n <= 128, 0 <= idx < 2086 and no label twice in one
    position for the first n entries, prob finite in float32, z in {-1, 0, 1}."""
    boards, n, idx, prob, z = (np.asarray(a) for a in (tb.boards, tb.n, tb.idx, tb.prob, tb.z))
    L = boards.shape[0] if boards.ndim == 2 else -1
    if boards.shape != (L, NSQ) or n.shape != (L,) or idx.shape != (L, MAXCHILD) or prob.shape != (L, MAXCHILD) or z.shape != (L,):
        raise ValueError("records must be boards [L,90], n [L], idx [L,128], prob [L,128], z [L]")
    if L == 0:
        return
    if not (np.issubdtype(boards.dtype, np.integer) and boards.min() >= 0 and boards.max() <= 14):
        raise ValueError("piece code outside 0..14")
    if not np.issubdtype(n.dtype, np.integer) or n.min() < 0 or n.max() > MAXCHILD:
        raise ValueError("move count outside 0..%d" % MAXCHILD)
    valid = np.arange(MAXCHILD)[None, :] < n[:, None]
    iv = idx[valid].astype(np.int64)
    if len(iv) and (iv.min() < 0 or iv.max() >= NLABEL):
        raise ValueError("label index outside 0..%d" % (NLABEL - 1))
    key = np.nonzero(valid)[0] * NLABEL + iv
    if len(np.unique(key)) != len(key):
        raise ValueError("a label appears twice in one position")
    with np.errstate(over="ignore", invalid="ignore"):
        if not np.isfinite(prob[valid].astype(np.float32)).all():
            raise ValueError("probability not finite in float32")
    if not np.isin(z, (-1.0, 0.0, 1.0)).all():
        raise ValueError("z outside {-1, 0, 1}")


class RingIndex:
    """Host bookkeeping of a ring of `capacity` slots that behaves like deque(maxlen=capacity): logical position 0 is the oldest
    surviving item, and adding k > capacity items keeps the last capacity of them."""

    def __init__(self, capacity):
        if int(capacity) <= 0:
            raise ValueError("capacity must be positive")
        self.capacity, self.head, self.size = int(capacity), 0, 0      # head: the next slot written

    def __len__(self):
        return self.size

    def add(self, k):
        """Reserve slots for k new items -> (first item kept, slots [k - first]): items [first, k) go to those slots in order."""
        first = max(0, int(k) - self.capacity)
        slots = (self.head + np.arange(int(k) - first)) % self.capacity
        self.head = int((self.head + len(slots)) % self.capacity)
        self.size = min(self.capacity, self.size + len(slots))
        return first, slots

    def slots(self, logical):
        """Ring slots of logical positions (0 = oldest)."""
        return (self.head - self.size + np.asarray(logical, dtype=np.int64)) % self.capacity

    def sample_rows(self, rng, k):
        """The slots of rng.sample(range(len), k): for the same random.Random state, the rows random.sample(deque, k) would pick."""
        return self.slots(rng.sample(range(self.size), k))


class ReplayBuffer:
    """The replay deque of main.py:1138 (deque(maxlen=buffer_size)) as a ring of device arrays, one per field:
    boards u8 [cap,90] (side-to-move canonical), n u8 [cap], idx i16 [cap,128], prob f32 [cap,128], z f32 [cap]."""

    def __init__(self, capacity=10000, device=None):
        self.ring = RingIndex(capacity)
        self.capacity = self.ring.capacity
        self.device = torch.device("cuda", torch.cuda.current_device() if device is None else device)
        cap, dev = self.capacity, self.device
        self.boards = torch.zeros((cap, NSQ), dtype=torch.uint8, device=dev)
        self.n = torch.zeros((cap,), dtype=torch.uint8, device=dev)
        self.idx = torch.zeros((cap, MAXCHILD), dtype=torch.int16, device=dev)
        self.prob = torch.zeros((cap, MAXCHILD), dtype=torch.float32, device=dev)
        self.z = torch.zeros((cap,), dtype=torch.float32, device=dev)
        self.added = 0                                  # positions ever added

    def __len__(self):
        return len(self.ring)

    def add(self, tb):
        """Append the tuples of a TupleBatch (distributed.pack_records / AsyncTupleGather.finish), oldest first; validated on the
        host (validate_tuples), then copied to the device.  prob is rounded to float32 as train_step's np.asarray(probs, float32)."""
        validate_tuples(tb)
        k = len(tb)
        self.added += k
        first, slots = self.ring.add(k)
        if not len(slots):
            return
        dev = self.device
        sl = torch.from_numpy(slots).to(dev)
        for dst, src in ((self.boards, tb.boards.astype(np.uint8)), (self.n, tb.n.astype(np.uint8)), (self.idx, tb.idx.astype(np.int16)),
                         (self.prob, tb.prob.astype(np.float32)), (self.z, tb.z.astype(np.float32))):
            dst.index_copy_(0, sl, torch.from_numpy(np.ascontiguousarray(src[first:])).to(dev))

    def sample_rows(self, rng, k):
        return self.ring.sample_rows(rng, k)

    def batch(self, rows, mirror=None):
        """-> (planes f32 [k,9,10,14], pi f32 [k,2086], z f32 [k,1]) on the device for ring slots `rows` (cz_replay_batch).
        mirror: k flags or None; a flagged row is mirrored left to right (board and move labels)."""
        rows = np.asarray(rows)
        if rows.ndim != 1 or not np.issubdtype(rows.dtype, np.integer):
            raise ValueError("rows must be a 1-d integer array")
        k = len(rows)
        if k and (rows.min() < 0 or rows.max() >= len(self)):
            raise ValueError("row index outside 0..%d" % (len(self) - 1))
        dev = self.device
        planes = torch.empty((k, 9, 10, 14), dtype=torch.float32, device=dev)
        pi = torch.empty((k, NLABEL), dtype=torch.float32, device=dev)
        z = torch.empty((k, 1), dtype=torch.float32, device=dev)
        if k == 0:
            return planes, pi, z
        rows_d = torch.from_numpy(rows.astype(np.int32)).to(dev)
        mir_d = None
        if mirror is not None:
            mirror = np.asarray(mirror)
            if mirror.shape != (k,):
                raise ValueError("mirror must hold one flag per row")
            mir_d = torch.from_numpy((mirror != 0).astype(np.uint8)).to(dev)
        rc = lib().cz_replay_batch(self.boards.data_ptr(), self.n.data_ptr(), self.idx.data_ptr(), self.prob.data_ptr(), self.z.data_ptr(),
                                   self.capacity, rows_d.data_ptr(), None if mir_d is None else mir_d.data_ptr(), k,
                                   planes.data_ptr(), pi.data_ptr(), z.data_ptr(), C.c_void_p(torch.cuda.current_stream(dev).cuda_stream))
        check(rc, "cz_replay_batch")
        return planes, pi, z

    def save(self, path):
        """np.savez of the ring (write + rename: never a half-written file); read back without pickle by load()."""
        _savez(path, capacity=self.capacity, head=self.ring.head, size=self.ring.size, added=self.added, boards=self.boards.cpu().numpy(),
               n=self.n.cpu().numpy(), idx=self.idx.cpu().numpy(), prob=self.prob.cpu().numpy(), z=self.z.cpu().numpy())

    def load(self, path):
        with np.load(path, allow_pickle=False) as d:
            if int(d["capacity"]) != self.capacity:
                raise ValueError("replay file holds a ring of %d, this buffer has %d" % (int(d["capacity"]), self.capacity))
            size, head = int(d["size"]), int(d["head"])
            if not (0 <= size <= self.capacity and 0 <= head < self.capacity):
                raise ValueError("replay file: bad ring position")
            a = {k: d[k] for k in ("boards", "n", "idx", "prob", "z")}
            added = int(d["added"])
        if a["boards"].shape[0] != self.capacity:
            raise ValueError("replay file: arrays do not match the ring capacity")
        validate_tuples(types.SimpleNamespace(**a))              # (unused slots are zero records, which pass)
        for k, v in a.items():
            getattr(self, k).copy_(torch.from_numpy(np.ascontiguousarray(v)))
        self.ring.head, self.ring.size, self.added = head, size, added


def _savez(path, **arrays):
    tmp = path + ".tmp"
    with open(tmp, "wb") as f:
        np.savez(f, **arrays)
    os.replace(tmp, path)


# ---- networks ------------------------------------------------------------------------------------------------------------
def _save_network(net, directory):
    """policy_value_network.save (weights, optimizer, global_step) into `directory`."""
    prev, net.save_dir = net.save_dir, directory
    try:
        return net.save(net.global_step)
    finally:
        net.save_dir = prev


def _restore_network(net, directory):
    idx = os.path.join(directory, "checkpoint")
    with open(idx) as f:
        name = f.read().strip()
    net.restore(os.path.join(directory, name))


def _clone_network(net, save_dir):
    """A second policy_value_network with the weights of `net` (same blocks, precision, device)."""
    from .net import policy_value_network
    with contextlib.redirect_stdout(sys.stderr), tempfile.TemporaryDirectory() as d:
        other = policy_value_network(len(net.net.blocks), precision=net.precision, device=net.device.index, seed=None,
                                     update_moving_stats=net.net.bn_in.update, save_dir=d)
    other.net.load_state_dict(net.net.state_dict())
    other.weights_version += 1
    other.save_dir = save_dir
    return other


def _num(v):
    """JSON-safe number: non-finite values as strings (a KL row sum can be -inf, see policy_kl)."""
    v = float(v)
    return v if math.isfinite(v) else str(v)


class Trainer:
    """AlphaZero's loop on one GPU with the reference's training rule.

    One ply (ply()):
      1. SelfPlay.step() over n_games concurrent games (auto reset; finished games keep their records);
      2. the finished games -> pack_records -> TupleBatch -> ReplayBuffer.add;
      3. for every finished game, in slot order, once the buffer holds more than batch_size positions: updates_per_game x
         policy_update() -- the reference's one update per game (main.py:1240-1242);
      4. with eval_every > 0, every eval_every finished games: arena.Match(candidate, best, eval_games, eval_playouts), and on
         promote(gate_threshold) the candidate's weights are copied into `best`.
    With eval_every = 0 self-play uses the trained network itself, as run() does.  With a gate, self-play uses `best` (a second
    policy_value_network; its plans re-fold the new weights in place after a promotion) and `network` is the candidate.

    policy_update() is cchess_main.policy_update (main.py:1157-1205) on the device: the same random.sample rows (sample_rows on the
    Trainer's random.Random), the mini-batch assembled by cz_replay_batch, old logits from the network's inference plan, up to
    `epochs` train steps with the early stop at kl > 4 kl_targ, the lr_multiplier rule and the explained variance.  One deliberate
    difference: the reference saves a checkpoint after every update (main.py:1189); the Trainer saves every `checkpoint_every`
    updates (0 = never) into the network's save_dir.  mirror=True flips a random half of every mini-batch left to right (the
    reference does no augmentation).

    save(dir) / load(dir) keep everything a run needs to continue: the network(s) with their optimizer state, the replay buffer,
    the sampler's random state, every game slot's MT19937 states (move choice and, with root noise, the noise stream), lr_multiplier,
    the counters and the games in flight (SelfPlay.save_games: the engine's trees and each slot's unfinished record), so a resumed
    run plays on exactly as the uninterrupted one.  load refuses a run saved with other rules, another root noise setting or
    other priors.  A directory saved without games.npz resumes with fresh games in every slot (drawing from the restored
    per-slot streams)."""

    def __init__(self, network, n_games, playouts, search_threads=1, batch_size=512, buffer_size=10000, epochs=5, kl_targ=0.025,
                 learning_rate=1e-3, updates_per_game=1, mirror=False, eval_every=0, eval_games=10, eval_playouts=None,
                 gate_threshold=0.55, checkpoint_every=100, seed=0, arena_words=1 << 20, best=None, rules="reference", root_noise=None,
                 priors="reference"):
        """rules: 'reference' or 'strict' -- self-play and the gate's matches search strictly legal moves only and a side without
        one is mated (the network learns the full rules of xiangqi); strict rules need search_threads = 1.  root_noise: None or
        (eps, alpha) -- Dirichlet noise on the root priors of every self-play search (SelfPlay root_noise); the gate's matches
        stay noise-free.  priors: 'reference' or 'softmax' -- how self-play and the gate's matches turn the network's logits into
        priors (SelfPlay priors)."""
        from .engine import check_priors, check_rules
        from .selfplay import check_root_noise, network_selfplay
        if eval_every and (eval_games <= 0 or eval_games % 2):
            raise ValueError("eval_games must be a positive even number (colour-swapped pairs)")
        self.rules = check_rules(rules, search_threads)
        self.root_noise = check_root_noise(root_noise)
        self.priors = check_priors(priors)
        self.network = network
        self.n_games, self.playouts, self.search_threads = int(n_games), playouts, int(search_threads)
        self.batch_size, self.epochs, self.kl_targ = int(batch_size), int(epochs), kl_targ
        self.learning_rate, self.lr_multiplier = learning_rate, 1.0
        self.updates_per_game, self.mirror = int(updates_per_game), bool(mirror)
        self.eval_every, self.eval_games = int(eval_every), int(eval_games)
        self.eval_playouts = playouts if eval_playouts is None else eval_playouts
        self.gate_threshold, self.checkpoint_every = gate_threshold, int(checkpoint_every)
        self.seed, self.arena_words = int(seed), arena_words
        self.rng = random.Random(self.seed)
        self.best = None
        if self.eval_every > 0:
            self.best = best if best is not None else _clone_network(network, os.path.join(network.save_dir, "best"))
        self.buffer = ReplayBuffer(buffer_size, network.device.index)
        self.sp = network_selfplay(self.best or network, self.n_games, playouts, seeds=[self.seed * self.n_games + g for g in range(self.n_games)],
                                   search_threads=self.search_threads, arena_words=arena_words, auto_reset=True, keep_records=True,
                                   rules=self.rules, root_noise=self.root_noise, priors=self.priors)
        self.sp.capture_graph()
        self.games = self.positions = self.updates = self.train_steps = self.promotions = self.gates = self.plies = 0
        self.next_gate = self.eval_every
        self.seconds = dict(selfplay=0.0, ingest=0.0, train=0.0, gate=0.0)
        self.last = None            # the last policy_update's statistics
        self.last_gate = None       # the last gate's MatchResult.to_json(games=False), parsed

    # -- training ---------------------------------------------------------------------------------------------------------
    def _forward(self, x):
        """policy_value_network.forward on a device batch: the plan's logits (no softmax) and value, as host arrays."""
        net = self.network
        logits, value = net.plan()(x.to(net.nn_dtype))
        return logits.cpu().numpy(), value.reshape(-1, 1).cpu().numpy()

    def policy_update(self):
        """One update of main.py:1157-1205 on a mini-batch of batch_size buffer rows; returns its statistics."""
        net = self.network
        rows = self.buffer.sample_rows(self.rng, self.batch_size)
        mirror = None
        if self.mirror:
            bits = self.rng.getrandbits(len(rows))
            mirror = np.array([(bits >> i) & 1 for i in range(len(rows))], dtype=np.uint8)
        x, pi, z = self.buffer.batch(rows, mirror)
        old_probs, old_v = self._forward(x)
        kl, loss, accuracy, new_v = 0.0, 0.0, 0.0, old_v
        steps = 0
        for _ in range(self.epochs):
            accuracy, loss, _ = net.train_step_device(x, pi, z, self.learning_rate * self.lr_multiplier)
            steps += 1
            new_probs, new_v = self._forward(x)
            kl = policy_kl(old_probs, new_probs)
            if kl > self.kl_targ * 4:
                break
        self.lr_multiplier = next_lr_multiplier(kl, self.kl_targ, self.lr_multiplier)
        wb = z.cpu().numpy().astype(np.float64)
        self.updates += 1
        self.train_steps += steps
        self.last = dict(rows=rows, steps=steps, loss=loss, accuracy=accuracy, kl=kl, lr_multiplier=self.lr_multiplier,
                         explained_var_old=explained_variance(wb, old_v), explained_var_new=explained_variance(wb, new_v))
        if self.checkpoint_every and self.updates % self.checkpoint_every == 0:
            net.save(net.global_step)
        return self.last

    # -- gate ---------------------------------------------------------------------------------------------------------------
    def gate(self):
        """arena.Match(candidate, best); promotes on MatchResult.promote(gate_threshold).  Returns the MatchResult."""
        from .arena import Match
        g0 = self.gates * self.eval_games
        r = Match(self.network, self.best, self.eval_games, self.eval_playouts, search_threads=self.search_threads,
                  seeds=range(g0, g0 + self.eval_games), arena_words=self.arena_words, rules=self.rules,
                  priors=self.priors).run()
        self.gates += 1
        self.last_gate = json.loads(r.to_json(self.gate_threshold, games=False))
        if r.promote(self.gate_threshold):
            self.promote()
        return r

    def promote(self):
        """best <- candidate: weights copied (the self-play plans re-fold them in place before the next search) and saved."""
        with torch.no_grad():
            self.best.net.load_state_dict(self.network.net.state_dict())
        self.best.weights_version += 1
        self.best.global_step = self.network.global_step
        self.best.save(self.best.global_step)
        self.promotions += 1

    # -- the loop -----------------------------------------------------------------------------------------------------------
    def ply(self):
        t0 = time.perf_counter()
        self.sp.step()
        t1 = time.perf_counter()
        finished = self.sp.pop_finished()
        if finished:
            buf, k, _ = pack_records([rec for _, rec in finished])
            self.buffer.add(TupleBatch(buf))
            self.games += len(finished)
            self.positions += k
        torch.cuda.synchronize(self.network.device)
        t2 = time.perf_counter()
        for _ in finished:
            if len(self.buffer) > self.batch_size:
                for _ in range(self.updates_per_game):
                    self.policy_update()
        t3 = time.perf_counter()
        while self.eval_every > 0 and self.games >= self.next_gate:
            self.gate()
            self.next_gate += self.eval_every
        t4 = time.perf_counter()
        self.plies += 1
        for key, dt in (("selfplay", t1 - t0), ("ingest", t2 - t1), ("train", t3 - t2), ("gate", t4 - t3)):
            self.seconds[key] += dt
        return len(finished)

    def report(self):
        """One JSON-ready dict: progress, the last update's statistics, the wall-time split and the last gate result."""
        last = self.last or {}
        d = dict(plies=self.plies, games=self.games, positions=self.positions, buffer=len(self.buffer), buffer_capacity=self.buffer.capacity,
                 updates=self.updates, train_steps=self.train_steps, global_step=self.network.global_step, promotions=self.promotions)
        for k in ("loss", "accuracy", "kl", "lr_multiplier", "explained_var_old", "explained_var_new"):
            d[k] = _num(last[k]) if k in last else None
        d["seconds"] = {k: round(v, 4) for k, v in self.seconds.items()}
        d["gate"] = self.last_gate
        return d

    def run(self, max_games=None, max_plies=None, report_every=10, report=None):
        """Plies until max_games games have finished or max_plies plies were played (None: no limit); report(dict) every
        report_every plies and once at the end."""
        report = report or (lambda d: print(json.dumps(d), flush=True))
        n = 0
        while (max_games is None or self.games < max_games) and (max_plies is None or n < max_plies):
            self.ply()
            n += 1
            if report_every and n % report_every == 0:
                report(self.report())
        report(self.report())

    # -- resume -------------------------------------------------------------------------------------------------------------
    def save(self, directory):
        """Everything a run needs to continue (see the class docstring) into `directory`."""
        os.makedirs(directory, exist_ok=True)
        _save_network(self.network, os.path.join(directory, "network"))
        if self.best is not None:
            _save_network(self.best, os.path.join(directory, "best"))
        self.buffer.save(os.path.join(directory, "replay.npz"))
        version, internal, gauss = self.rng.getstate()
        # root_noise: [eps, alpha], or empty when off; the noise streams' states go with it
        noise = dict(root_noise=np.asarray(self.root_noise or (), dtype=np.float64))
        if self.root_noise is not None:
            noise["noise_mt"] = self.sp._noise_mt
        priors = getattr(self, "priors", "reference")
        if priors != "reference":                          # (absent: reference priors, so the default run's file is unchanged)
            noise["priors"] = np.asarray(priors)
        _savez(os.path.join(directory, "trainer.npz"), rng_version=version, rng_internal=np.asarray(internal, dtype=np.uint32),
               rng_gauss=np.float64(0.0 if gauss is None else gauss), rng_has_gauss=gauss is not None, mt=self.sp._mt, **noise,
               lr_multiplier=self.lr_multiplier, next_gate=self.next_gate, rules=np.asarray(self.rules),
               counters=np.asarray([self.games, self.positions, self.updates, self.train_steps, self.promotions, self.gates, self.plies],
                                   dtype=np.int64))
        self.sp.save_games(os.path.join(directory, "games.npz"))

    def load(self, directory):
        """Restore what save() wrote, the games in flight included; without games.npz every slot starts a fresh game."""
        with np.load(os.path.join(directory, "trainer.npz"), allow_pickle=False) as d:
            if d["mt"].shape != self.sp._mt.shape:
                raise ValueError("saved run has %d game slots, this Trainer %d" % (d["mt"].shape[0], self.n_games))
            saved = str(d["rules"]) if "rules" in d.files else "reference"          # (runs saved before the rules choice existed)
            if saved != self.rules:
                raise ValueError("saved run plays by the %r rules, this Trainer by %r" % (saved, self.rules))
            rn = d["root_noise"] if "root_noise" in d.files else np.zeros(0)    # (runs saved before root noise existed: off)
            saved = tuple(float(v) for v in rn) if rn.size else None
            if saved != self.root_noise:
                raise ValueError("saved run has root noise %r, this Trainer %r" % (saved, self.root_noise))
            saved, priors = (str(d["priors"]) if "priors" in d.files else "reference"), getattr(self, "priors", "reference")
            if saved != priors:
                raise ValueError("saved run uses the %r priors, this Trainer %r" % (saved, priors))
            noise_mt = d["noise_mt"].copy() if self.root_noise is not None else None
            gauss = float(d["rng_gauss"]) if bool(d["rng_has_gauss"]) else None
            self.rng.setstate((int(d["rng_version"]), tuple(int(v) for v in d["rng_internal"]), gauss))
            mt = d["mt"].copy()
            self.lr_multiplier, self.next_gate = float(d["lr_multiplier"]), int(d["next_gate"])
            (self.games, self.positions, self.updates, self.train_steps, self.promotions, self.gates,
             self.plies) = (int(v) for v in d["counters"])
        _restore_network(self.network, os.path.join(directory, "network"))
        if self.best is not None:
            _restore_network(self.best, os.path.join(directory, "best"))
        self.buffer.load(os.path.join(directory, "replay.npz"))
        games = os.path.join(directory, "games.npz")
        if os.path.isfile(games):
            self.sp.load_games(games)
        else:
            self.sp.restart_games(mt, noise_mt)


def main(argv=None):
    ap = argparse.ArgumentParser(description="Train a policy-value network by batched self-play on one GPU; one JSON line per report.")
    ap.add_argument("--games", type=int, default=1024, help="concurrent self-play games")
    ap.add_argument("--playouts", type=int, default=400)
    ap.add_argument("--search-threads", type=int, default=1)
    ap.add_argument("--batch-size", type=int, default=512)
    ap.add_argument("--buffer-size", type=int, default=10000)
    ap.add_argument("--epochs", type=int, default=5)
    ap.add_argument("--learning-rate", type=float, default=1e-3)
    ap.add_argument("--updates-per-game", type=int, default=1)
    ap.add_argument("--res-block-nums", type=int, default=7)
    ap.add_argument("--precision", default="fp16", help="inference precision of self-play and of the KL forward passes")
    ap.add_argument("--eval-every", type=int, default=0, help="finished games between gates (0: no gate, self-play uses the trained network)")
    ap.add_argument("--eval-games", type=int, default=10)
    ap.add_argument("--eval-playouts", type=int, default=None)
    ap.add_argument("--gate-threshold", type=float, default=0.55)
    ap.add_argument("--checkpoint-every", type=int, default=100, help="updates between checkpoints (0: none)")
    ap.add_argument("--max-games", type=int, default=None)
    ap.add_argument("--max-plies", type=int, default=None)
    ap.add_argument("--report-every", type=int, default=10, help="plies between JSON lines")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--mirror", action="store_true", help="mirror a random half of every mini-batch left to right")
    ap.add_argument("--save-dir", required=True, help="checkpoints and the state a --resume continues from")
    ap.add_argument("--resume", action="store_true", help="continue the run saved in --save-dir")
    ap.add_argument("--rules", choices=("reference", "strict"), default="reference",
                    help="strict: search strictly legal moves only; a side without one is mated (needs --search-threads 1)")
    ap.add_argument("--root-noise", nargs=2, type=float, metavar=("EPS", "ALPHA"), default=None,
                    help="Dirichlet noise on the self-play root priors: P' = (1 - EPS) P + EPS Dir(ALPHA), e.g. 0.25 0.3")
    ap.add_argument("--priors", choices=("reference", "softmax"), default="reference",
                    help="softmax: self-play and the gate search with the softmax of the legal moves' logits as priors (reference: "
                         "logit / sum, the reference's expansion)")
    a = ap.parse_args(argv)
    from .net import policy_value_network
    out = sys.stdout
    with contextlib.redirect_stdout(sys.stderr):                    # library prints (checkpoint paths) stay off the JSON stream
        with tempfile.TemporaryDirectory() as d:                    # nothing is picked up implicitly from an old checkpoint index
            net = policy_value_network(a.res_block_nums, precision=a.precision, seed=a.seed, save_dir=d)
        net.save_dir = os.path.join(a.save_dir, "network")
        t = Trainer(net, a.games, a.playouts, search_threads=a.search_threads, batch_size=a.batch_size, buffer_size=a.buffer_size,
                    epochs=a.epochs, learning_rate=a.learning_rate, updates_per_game=a.updates_per_game, mirror=a.mirror,
                    eval_every=a.eval_every, eval_games=a.eval_games, eval_playouts=a.eval_playouts, gate_threshold=a.gate_threshold,
                    checkpoint_every=a.checkpoint_every, seed=a.seed, rules=a.rules, root_noise=a.root_noise,
                    priors=a.priors)
        if t.best is not None:
            t.best.save_dir = os.path.join(a.save_dir, "best")
        if a.resume and os.path.isfile(os.path.join(a.save_dir, "trainer.npz")):
            t.load(a.save_dir)
        t.run(a.max_games, a.max_plies, a.report_every, report=lambda r: print(json.dumps(r), file=out, flush=True))
        t.save(a.save_dir)
    return t


if __name__ == "__main__":
    main()
