"""An independent pure-Python restatement of pixo's LZ77 parse and of huffman::build_codes, for small inputs.  It is
written from pixo's source (src/compress/lz77.rs:329-876,1399-1480 and src/compress/huffman.rs:30-205), not from
oracle/png_deflate.c, and checks that oracle token for token and length for length.  Each branch the tests need to
reach is recorded in `events`, so a test can assert that its input really took it.

lz77(data, level) -> (tokens as pixo's packed u32 list, events: set of str)
build_lengths(freqs, max_len) -> (lengths list, events)
"""
from __future__ import annotations

MAX_DISTANCE, MAX_MATCH, MIN_MATCH = 32768, 258, 3
# config_for_level: (max_chain_length, max_search_depth, nice_length, lazy, use_ht)
LEVELS = {1: (4, 4, 32, None, True), 2: (8, 6, 10, None, False), 3: (16, 12, 14, None, False),
          4: (32, 16, 30, None, False), 5: (64, 16, 30, "lazy", False), 6: (128, 35, 65, "lazy", False),
          7: (256, 100, 130, "lazy", False), 8: (1024, 300, 258, "lazy2", False),
          9: (4096, 600, 258, "lazy2", False)}
M32 = 0xFFFFFFFF


class _Parser:
    def __init__(self, data: bytes, level: int):
        self.d, self.n = data, len(data)
        self.chain, self.depth, self.nice, self.lazy, self.ht = LEVELS[level]
        self.head, self.head3, self.prev = {}, {}, {}
        self.buckets = {}
        self.ev = set()

    def _u32(self, p, k=4):
        return int.from_bytes(self.d[p:p + k].ljust(4, b"\0"), "little")

    def hash4(self, p):
        if p + 3 >= self.n:
            self.ev.add("hash4_zero")
            return 0
        return ((self._u32(p) * 0x1E35A7BD) & M32) >> 16 & 0xFFFF

    def hash3(self, p):
        if p + 2 >= self.n:
            return 0
        return ((self._u32(p, 3) * 0x1E35A7BD) & M32) >> 17 & 0x7FFF

    def hash4_ht(self, p):
        if p + 3 >= self.n:
            return 0
        return ((self._u32(p) * 0x1E35A7BD) & M32) >> 17 & 0x7FFF

    def match_length(self, a, b):
        m = min(self.n - b, MAX_MATCH)
        k = 0
        while k < m and self.d[a + k] == self.d[b + k]:
            k += 1
        return k

    def update_hash(self, p):
        if p + 3 >= self.n:
            return
        self.head3[self.hash3(p)] = p
        h = self.hash4(p)
        self.prev[p % MAX_DISTANCE] = self.head.get(h, -1)
        self.head[h] = p

    def run_length(self, p):
        m = min(self.n - p, MAX_MATCH)
        k = 1
        while k < m and self.d[p + k] == self.d[p]:
            k += 1
        return k

    def accept(self, length, dist, best, best_d, minm):
        if length < minm:
            return False
        if length == 3 and dist > 8192:
            self.ev.add("gate_8192")
            return False
        return length > best or (length == best and dist < best_d)

    def find(self, pos, chain, minm):
        d = self.d
        if pos + MIN_MATCH > self.n:
            return None
        run = self.run_length(pos)
        is_run = run >= minm and pos >= 1 and d[pos - 1] == d[pos]
        if is_run and (run >= self.nice or run >= MAX_MATCH):
            self.ev.add("run_nice")
            return min(run, MAX_MATCH), 1
        best, best_d = max(minm - 1, 0), 0
        if is_run:
            best, best_d = run, 1
        c3 = self.head3.get(self.hash3(pos), -1)
        if c3 >= 0:
            dist = pos - c3
            if dist != 0 and dist <= MAX_DISTANCE and d[pos:pos + 3] == d[c3:c3 + 3]:
                length = min(self.match_length(c3, pos), MAX_MATCH)
                if self.accept(length, dist, best, best_d, minm):
                    best, best_d = length, dist
                    if best >= self.nice:
                        self.ev.add("nice_exit")
                        return best, best_d
        cp = self.head.get(self.hash4(pos), -1)
        maxd = min(pos, MAX_DISTANCE)
        prefix = d[pos:pos + 4] if pos + 4 <= self.n else None
        left = chain
        while cp >= 0 and left > 0:
            mp = cp
            dist = pos - mp
            cp = self.prev.get(mp % MAX_DISTANCE, -1)
            left -= 1
            if dist == 0:
                continue
            if dist > maxd:
                self.ev.add("window_break")
                break
            if prefix is not None and mp + 4 <= self.n and d[mp:mp + 4] != prefix:
                continue
            length = self.match_length(mp, pos)
            if self.accept(length, dist, best, best_d, minm):
                best, best_d = length, dist
                if length >= MAX_MATCH or best >= self.nice:
                    self.ev.add("nice_exit")
                    break
        return (best, best_d) if best >= minm else None

    def find_ht(self, pos, minm):
        if pos + MIN_MATCH > self.n:
            return None
        h = self.hash4_ht(pos)
        c0, c1 = self.buckets.get(h, (-1, -1))
        self.buckets[h] = (pos, c0)
        self.ev.add("ht")
        best, best_d = max(minm - 1, 0), 0
        for c in (c0, c1):
            if c < 0:
                continue
            dist = pos - c
            if dist == 0 or dist > MAX_DISTANCE or self.d[pos:pos + 3] != self.d[c:c + 3]:
                continue
            length = min(self.match_length(c, pos), MAX_MATCH)
            if length < minm:
                continue
            if length == 3 and dist > 8192:
                self.ev.add("gate_8192")
                continue
            if length > best:
                best, best_d = length, dist
                if best >= self.nice:
                    self.ev.add("nice_exit")
                    break
        return (best, best_d) if best >= minm else None

    def min_match(self):
        used = len(set(self.d[:4096]))
        if self.depth <= 4:
            return MIN_MATCH
        m = MIN_MATCH
        if used > 32:
            m = 4
        if used > 64 and self.depth >= 10:
            m = 5
        if used > 96 and self.depth >= 20:
            m = 6
        return m

    def after_match(self, pos, length, dist):
        if dist == 1:
            self.ev.add("run_dist1")
            self.update_hash(pos)
            self.update_hash(pos + length - 1)
        else:
            for i in range(length):
                self.update_hash(pos + i)
        if pos + length == self.n:
            self.ev.add("tail_match")

    def parse(self):
        d, n, out = self.d, self.n, []
        if n == 0:
            return out
        minm = self.min_match()
        pos = streak = probe = updates = 0
        incompressible = False
        pending = None
        lit = lambda b: out.append(0x80000000 | b)
        mat = lambda length, dist: out.append((dist - 1) << 16 | length)
        while pos < n:
            if incompressible:
                if probe >= 256:
                    probe = 0
                    m = self.find(pos, min(1, self.depth), minm)
                    if m:
                        self.ev.add("probe_exit")
                        incompressible, streak = False, 0
                        mat(*m)
                        self.after_match(pos, *m)
                        pos += m[0]
                        continue
                lit(d[pos])
                updates += 1
                if updates >= 64:
                    self.update_hash(pos)
                    updates = 0
                pos += 1
                streak += 1
                probe += 1
                continue
            chain = self.chain
            if streak >= 512:
                incompressible, probe, chain = True, 0, 1
            if pending:
                m, pending = pending, None
            elif self.ht:
                m = self.find_ht(pos, minm)
            else:
                m = self.find(pos, min(chain, self.depth), minm)
            if m:
                length, dist = m
                streak, incompressible, probe = 0, False, 0
                if self.lazy and length < self.nice and length < 16 and pos + 1 < n:
                    self.update_hash(pos)
                    nxt_chain = max(chain // 2, 1) if self.lazy == "lazy2" else chain
                    nm = self.find_ht(pos + 1, minm) if self.ht else self.find(pos + 1, min(nxt_chain, self.depth), minm)
                    if nm and (nm[0] >= length + 3 or nm[0] >= self.nice):
                        self.ev.add(self.lazy + "_defer")
                        lit(d[pos])
                        pending = nm
                        pos += 1
                        continue
                mat(length, dist)
                self.after_match(pos, length, dist)
                pos += length
            else:
                streak += 1
                if streak >= 512:
                    self.ev.add("incompressible_enter")
                    incompressible, probe, updates = True, 0, 0
                lit(d[pos])
                self.update_hash(pos)
                pos += 1
        return out


def lz77(data: bytes, level: int):
    p = _Parser(bytes(data), level)
    return p.parse(), p.ev


def is_high_entropy_data(data: bytes):
    """is_high_entropy_data (deflate.rs:1108-1145): (fires, collisions).  Streams under 4 096 bytes never fire; the
    first min(n, 8 192) bytes' 4-grams are hashed into 4 096 slots, and the bail fires when the share of 4-grams whose
    slot was already taken is below 5 %, divided in f32 (`collisions as f32 / total as f32 < 0.05`)."""
    import numpy as np
    if len(data) < 4096:
        return False, 0
    sample = bytes(data[:8192])
    seen, coll = set(), 0
    for i in range(len(sample) - 3):
        h = ((int.from_bytes(sample[i:i + 4], "little") * 0x1E35A7BD) & M32) >> 20 & 4095
        coll += h in seen
        seen.add(h)
    return bool(np.float32(coll) / np.float32(len(sample) - 3) < np.float32(0.05)), coll


# ---- build_codes with Rust's BinaryHeap<Reverse<Node>> ---------------------------------------------------------

def _key(node):
    """Node's Ord: (frequency, Option<symbol>) with None below every Some."""
    f, sym = node[0], node[1]
    return (f, -1 if sym is None else sym)


class _RustHeap:
    """std::collections::BinaryHeap of Reverse<Node>: a max-heap, so 'greater' is the smaller node."""

    def __init__(self, items, ev):
        self.h, self.ev = list(items), ev
        for k in range(len(self.h) // 2 - 1, -1, -1):   # rebuild
            self._sift_down_range(k, len(self.h))

    def _le(self, a, b):   # Reverse(a) <= Reverse(b)
        ka, kb = _key(a), _key(b)
        if ka == kb and a[1] is None:
            self.ev.add("internal_tie")
        return kb <= ka

    def _lt(self, a, b):
        return _key(b) < _key(a)

    def _sift_up(self, start, pos):
        e = self.h[pos]
        while pos > start:
            parent = (pos - 1) // 2
            if self._le(e, self.h[parent]):
                break
            self.h[pos] = self.h[parent]
            pos = parent
        self.h[pos] = e

    def _sift_down_range(self, pos, end):
        e = self.h[pos]
        child = 2 * pos + 1
        while child <= end - 2:
            if self._le(self.h[child], self.h[child + 1]):
                child += 1
            if self._le(self.h[child], e):   # e >= child
                self.h[pos] = e
                return
            self.h[pos] = self.h[child]
            pos, child = child, 2 * child + 1
        if child == end - 1 and self._lt(e, self.h[child]):
            self.h[pos] = self.h[child]
            pos = child
        self.h[pos] = e

    def pop(self):
        item = self.h.pop()
        if self.h:
            item, self.h[0] = self.h[0], item
            end, pos, child = len(self.h), 0, 1
            e = self.h[0]
            while child <= end - 2:
                if self._le(self.h[child], self.h[child + 1]):
                    child += 1
                self.h[pos] = self.h[child]
                pos, child = child, 2 * child + 1
            if child == end - 1:
                self.h[pos] = self.h[child]
                pos = child
            self.h[pos] = e
            self._sift_up(0, pos)
        return item

    def push(self, x):
        self.h.append(x)
        self._sift_up(0, len(self.h) - 1)


def _depths(node, depth, out):
    if node[1] is not None:
        out[node[1]] = max(depth, 1)
    else:
        _depths(node[2], depth + 1, out)
        _depths(node[3], depth + 1, out)


def _limit(lengths, max_len, ev):
    if not any(x > max_len for x in lengths):
        return
    ev.add(f"limit_{max_len}")
    lengths[:] = [min(x, max_len) for x in lengths]
    lim = 1 << max_len
    k = sum(1 << (max_len - x) for x in lengths if x)
    while k > lim:
        cand = [(x, i) for i, x in enumerate(lengths) if 0 < x < max_len]
        if not cand:
            break
        x, i = min(cand)   # the shortest, first in symbol order
        k += (1 << (max_len - x - 1)) - (1 << (max_len - x))
        lengths[i] += 1
    while k < lim:
        best_i, best_l = None, 0
        for i, x in enumerate(lengths):
            if x > 1 and x > best_l:
                best_i, best_l = i, x
        if best_i is None:
            break
        new_k = k - (1 << (max_len - best_l)) + (1 << (max_len - best_l + 1))
        if new_k > lim:
            break
        k = new_k
        lengths[best_i] -= 1


def build_lengths(freqs, max_len: int, tie_order: str = "rust"):
    """build_codes' code lengths.  tie_order 'fifo' pops equal nodes in insertion order instead of Rust's heap order
    (only for showing that the order matters)."""
    ev = set()
    n = len(freqs)
    nz = [(int(f), i, None, None) for i, f in enumerate(freqs) if f]
    lengths = [0] * n
    if not nz:
        return lengths, ev
    if len(nz) == 1:
        lengths[nz[0][1]] = 1
        return lengths, ev
    if tie_order == "rust":
        heap = _RustHeap(nz, ev)
        while len(heap.h) > 1:
            a, b = heap.pop(), heap.pop()
            heap.push((a[0] + b[0], None, a, b))
        root = heap.h[0]
    else:
        import heapq
        q = [(_key(x), i, x) for i, x in enumerate(nz)]
        heapq.heapify(q)
        c = len(q)
        while len(q) > 1:
            a, b = heapq.heappop(q)[2], heapq.heappop(q)[2]
            x = (a[0] + b[0], None, a, b)
            heapq.heappush(q, (_key(x), c, x))
            c += 1
        root = q[0][2]
    _depths(root, 0, lengths)
    _limit(lengths, max_len, ev)
    return lengths, ev
