"""Corpora that take the drain kernel off its staged fast path, with expected records from plain references.

drain3_kernel (beta9_b200/csrc/drain2.cuh) gets a warp-tile's bytes in one of four ways:
  1. the tile is contiguous in the ring and its 16-byte-aligned span fits the warp's stage buffer: one bulk copy;
  2. it is contiguous but does not fit: crc32 / json_sum stage each task on its own (stage_one_task), identity and
     vadd_f32 read the ring through generic pointers;
  3. a single task is larger than the stage buffer: every handler reads it from the ring;
  4. the tile's tasks are not contiguous (the tile spans two pushes, or a push that wrapped to the ring's start):
     one bulk copy per task (d3_stage_scattered), refused when the aligned spans add up to more than the buffer.
The stage buffer's size comes from the window (launch_drain3 in b9gpu.cu); `stage_cap` and `read_paths` restate that
choice so that a corpus can show which ways its tiles take, and `RingModel` restates ring_place.h so that a sequence of
pushes and drains can show where the ring wraps.

Every builder returns a `Corpus`: payloads plus, per task, the expected (status, result bytes) from a reference that
shares no code with the device or the oracle (json / zlib / numpy / sum), or None where only the oracle decides (lone
surrogates and invalid UTF-8, where Go's decoder and json.loads disagree)."""
from __future__ import annotations

import base64
import json
import zlib
from collections import deque
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Set, Tuple

import numpy as np

FRAME_PRE = b'{"args": ["'
FRAME_SUF = b'"], "kwargs": {}}'
COMPLETE = 0
T_OF = {"identity": 32, "crc32": 4, "vadd_f32": 32, "json_sum": 8}     # D3Cfg<H>::T
STAGE_MIN, STAGE_MAX = 1 << 10, 48 << 10

Want = Optional[Tuple[int, Optional[bytes]]]


@dataclass
class Corpus:
    handler: str
    payloads: List[bytes] = field(default_factory=list)
    want: List[Want] = field(default_factory=list)        # None: the oracle decides

    def add(self, payload: bytes, want: Want) -> None:
        self.payloads.append(payload)
        self.want.append(want)

    def extend(self, other: "Corpus") -> None:
        assert other.handler == self.handler
        self.payloads += other.payloads
        self.want += other.want

    @property
    def n(self) -> int:
        return len(self.payloads)


# ------------------------------------------------------------------ references
def decode_body(body: bytes) -> Optional[str]:
    """The Python string a JSON string body stands for, or None when it is not well-formed (invalid UTF-8, a lone
    surrogate): there Go's decoder substitutes U+FFFD and json.loads does not, so only the oracle can say."""
    try:
        s = json.loads(b'"' + body + b'"')
        s.encode("utf-8")
    except (ValueError, UnicodeError):
        return None
    return s


def ref_identity(s: str) -> Want:
    return COMPLETE, (json.dumps(s).encode() if s else None)


def ref_crc32(s: str) -> Want:
    c = zlib.crc32(s.encode("utf-8"))
    return COMPLETE, (str(c).encode() if c else None)


def ref_string(handler: str, body: bytes) -> Want:
    s = decode_body(body)
    if s is None:
        return None
    return ref_identity(s) if handler == "identity" else ref_crc32(s)


def framed(body: bytes) -> bytes:
    return FRAME_PRE + body + FRAME_SUF


def vadd_task(a: np.ndarray, b: np.ndarray) -> Tuple[bytes, Want]:
    """A vadd_f32 payload over two float32 vectors without NaN, and numpy's float32 sum re-encoded as the handler does."""
    assert a.dtype == np.float32 and b.dtype == np.float32 and a.size == b.size and a.size
    assert not (np.isnan(a).any() or np.isnan(b).any())
    arg = base64.b64encode(np.concatenate([a, b]).astype("<f4").tobytes()).decode()
    with np.errstate(all="ignore"):
        c = (a + b).astype("<f4")
    out = base64.b64encode(c.tobytes()).decode()
    return json.dumps({"args": [arg], "kwargs": {}}).encode(), (COMPLETE, json.dumps(out).encode())


def json_sum_task(values: List[int], pad: int = 0, ident: int = 0) -> Tuple[bytes, Want]:
    doc = {"id": ident, "values": values, "pad": "x" * pad}
    s = sum(values)
    return json.dumps({"args": [doc], "kwargs": {}}).encode(), (COMPLETE, str(s).encode() if s else None)


# ------------------------------------------------------------------ the kernel's staging decisions, restated
def tile_tasks(handler: str, n: int) -> int:
    """Tasks per warp-tile of a window of n tasks. json_sum takes 4 when the window has fewer than three 8-task tiles
    per resident warp; with at least one CTA per SM on at least 114 SMs that is certain below the bound asserted here."""
    if handler != "json_sum":
        return T_OF[handler]
    assert (n + 7) // 8 < 3 * 114 * 2, "json_sum window too large to know its tile size"
    return 4


def stage_cap(handler: str, n: int, in_bytes: int, max_len: int, override: int = 0) -> int:
    """The stage buffer per warp that launch_drain3 picks for a window of n tasks and in_bytes payload bytes whose
    pushes' longest task is max_len (B9_STAGE_BYTES = override)."""
    if override:
        return override
    tt = tile_tasks(handler, n)
    avg = in_bytes // n
    want = avg * tt * 27 // 20 + 768 if handler == "crc32" else avg * tt * 11 // 10 + 768
    cap = min(STAGE_MAX, max(STAGE_MIN, want))
    if handler != "crc32" and max_len:
        cap = min(cap, max(STAGE_MIN, max_len * tt + 32))
    return (cap + 127) & ~127


def read_paths(offs, lens, tt: int, in_cap: int) -> Dict[str, int]:
    """How drain3_kernel reads every task of a window (tasks at ring offsets `offs`): counts of tasks per way
    ("1" staged tile, "2" own stage, "3" larger than the stage, "4" scattered tile staged) and of scattered tiles
    refused ("4r") or contiguous tiles of exactly the buffer's size ("fit")."""
    offs = [int(o) for o in offs]
    lens = [int(x) for x in lens]
    c = {"1": 0, "2": 0, "3": 0, "4": 0, "4r": 0, "fit": 0}
    for t0 in range(0, len(offs), tt):
        o, ln = offs[t0:t0 + tt], lens[t0:t0 + tt]
        contig = all(o[i] == o[i - 1] + ln[i - 1] for i in range(1, len(o)))
        if contig:
            span = ((o[-1] + ln[-1] + 15) & ~15) - (o[0] & ~15)
            staged = span <= in_cap
            c["fit"] += span == in_cap
        else:
            total = sum(((a + b + 15) & ~15) - (a & ~15) for a, b in zip(o, ln) if b)
            staged = total <= in_cap
            c["4r"] += not staged
        for a, b in zip(o, ln):
            if staged:
                c["1" if contig else "4"] += 1
            else:
                c["2" if (a & 15) + b + 16 <= in_cap else "3"] += 1
    return c


SEG_ALIGN = 256


def ring_place(ring_bytes: int, have_segments: bool, oldest: int, wp: int, live_bytes: int, nbytes: int) -> Optional[int]:
    """b9_ring_place (beta9_b200/csrc/ring_place.h): where a push segment of nbytes goes, or None."""
    need = (nbytes + SEG_ALIGN - 1) & ~(SEG_ALIGN - 1)
    if need > ring_bytes:
        return None
    if not have_segments:
        return 0
    if live_bytes == 0:
        return wp if wp + need <= ring_bytes else 0
    if wp == oldest:
        return wp if need == 0 else None
    if wp > oldest:
        if wp + need <= ring_bytes:
            return wp
        return 0 if need <= oldest else None
    return wp if wp + need <= oldest else None


class RingModel:
    """The host's segment bookkeeping (b9gpu.cu: place_segment, the push, the fetch that frees drained segments)."""

    def __init__(self, ring_bytes: int):
        self.ring = ring_bytes
        self.segs: deque = deque()         # [start, task lengths, first undrained index]
        self.wp = 0

    def push(self, lens: List[int]) -> Optional[int]:
        nbytes = sum(lens)
        live = sum(sum(s[1]) for s in self.segs)
        start = ring_place(self.ring, bool(self.segs), self.segs[0][0] if self.segs else 0, self.wp, live, nbytes)
        if start is None:
            return None
        self.segs.append([start, list(lens), 0])
        self.wp = start + ((nbytes + SEG_ALIGN - 1) & ~(SEG_ALIGN - 1))
        return start

    def window(self, n: int):
        """Ring offsets and lengths of the next n pending tasks, and the longest task of the pushes they are in."""
        offs, lens, max_len = [], [], 0
        for start, ln, k in self.segs:
            if len(offs) == n:
                break
            pos = start + sum(ln[:k])
            max_len = max(max_len, max(ln))
            for x in ln[k:]:
                if len(offs) == n:
                    break
                offs.append(pos)
                lens.append(x)
                pos += x
        return offs, lens, max_len

    def pop(self, n: int) -> None:
        while n:
            s = self.segs[0]
            take = min(n, len(s[1]) - s[2])
            s[2] += take
            n -= take
            if s[2] == len(s[1]):
                self.segs.popleft()
        if not self.segs:
            self.wp = 0

    def depth(self) -> int:
        return sum(len(s[1]) - s[2] for s in self.segs)


# ------------------------------------------------------------------ lane-boundary strings
LANE_S = (1, 2, 5, 8, 33, 1000, 40000)              # S = ceil(n / 32): bytes of body per lane chunk
LANE_KS = (1, 15, 31)                               # lane chunks whose start k*S gets a unit nearby
LANE_D = range(-6, 7)                               # offsets of the unit's first byte from k*S
UNITS: Dict[str, bytes] = {
    "quote": b'\\"', "backslash": b"\\\\", "slash": b"\\/", "newline": b"\\n",
    "u_lower": b"\\u00e9", "u_upper": b"\\u00E9",                  # u_upper: same length, text rewritten
    "pair": b"\\ud83d\\ude00",
    "lone_high_pair": b"\\ud83d\\ud83d\\ude00",                    # a lone high surrogate, then a pair (oracle only)
    "utf8_2": "é".encode(), "utf8_3": "€".encode(), "utf8_4": "\U0001F600".encode(),
    "bs_then_u_text": b"\\\\ud83d\\ude00",                          # \\ then the text ud83d\ude00: a lone low surrogate (oracle only)
    "bs_then_u_plain": b"\\\\ud83d",                                # \\ then plain text ud83d
    "utf8_bad_cont": b"\xe2\x82",                                  # a 3-byte lead with one continuation (oracle only)
    "utf8_surrogate": b"\xed\xa0\x80",                             # an encoded surrogate (oracle only)
}
_PLAIN = np.frombuffer(b"abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789 .,;:-_=+*!?#()<>", np.uint8)


def plain_text(n: int, seed: int) -> bytes:
    return _PLAIN[np.random.default_rng(seed).integers(0, _PLAIN.size, size=n)].tobytes()


def _lane_placements():
    """(S, body bytes, {(unit, k, d)}) for every unit at every offset around lane starts 1, 15 and 31 where the unit fits
    in the body. Bodies have n = 32 * S bytes. For S <= 33 one placement per body; for larger S the three lane starts
    are far apart and one body carries the same (unit, d) at all three."""
    for S in LANE_S:
        n = 32 * S
        filler = plain_text(n, seed=S)
        for name, u in UNITS.items():
            for d in LANE_D:
                groups = [[k] for k in LANE_KS] if S <= 33 else [list(LANE_KS)]
                for ks in groups:
                    pos = [k * S + d for k in ks if 0 <= k * S + d and k * S + d + len(u) <= n]
                    if not pos:
                        continue
                    b = bytearray(filler)
                    for p in pos:
                        b[p:p + len(u)] = u
                    yield S, bytes(b), {(name, (p - d) // S, d) for p in pos}


def lane_coverage_expected() -> Set[Tuple[int, str, int, int]]:
    return {(S, name, k, d) for S in LANE_S for name, u in UNITS.items() for k in LANE_KS for d in LANE_D
            if 0 <= k * S + d and k * S + d + len(u) <= 32 * S}


def lane_boundary_strings(handler: str) -> Corpus:
    assert handler in ("identity", "crc32")
    c = Corpus(handler)
    covered = set()
    for S, body, placed in _lane_placements():
        assert -(-len(body) // 32) == S
        c.add(framed(body), ref_string(handler, body))
        covered |= {(S,) + p for p in placed}
    assert covered == lane_coverage_expected()
    # from S = 33 on every unit fits at every offset around every one of the three lane starts
    for S in LANE_S[4:]:
        assert {p[1:] for p in covered if p[0] == S} == {(name, k, d) for name in UNITS for k in LANE_KS for d in LANE_D}
    for S in LANE_S:
        n = 32 * S
        if S >= 33:
            # more than two upper-case-hex escapes in every lane chunk: json.dumps rewrites all of them (esc_emit_general)
            b = bytearray(plain_text(n, seed=7 * S))
            for lane in range(32):
                for j in range(3):
                    p = lane * S + 2 + 8 * j
                    b[p:p + 6] = b"\\u00C%d" % (j + 1)
            c.add(framed(bytes(b)), ref_string(handler, bytes(b)))
        # bodies whose json.dumps form has another length: raw UTF-8 and "\/" spread through every chunk
        rng = np.random.default_rng(11 * S)
        s = "".join(rng.choice(["a", "b", "Z", " ", "é", "€", "\U0001F600", "/", '"', "\n"], size=max(1, n // 3)))
        for body in (json.dumps(s, ensure_ascii=False)[1:-1].encode(), json.dumps(s)[1:-1].replace("/", "\\/").encode()):
            c.add(framed(body), ref_string(handler, body))
    return c


# ------------------------------------------------------------------ crc32's zero-shift levels
# A lane's shift is the number of decoded bytes after its chunk; for a plain body of n bytes, lane l's is
# n - min(n, (l + 1) * S). The bodies below set every bit 0..25 of some lane's shift. Bits 26..29 would need tasks of
# 64 MiB to 1 GiB and bits 30..31 cannot occur under the 1 GiB task limit: those levels are not reached here.
SHIFT_BITS = 26
SHIFT_N = (32, 33, 100, 1056, 3000, 32000, 100_000, 1_000_003, 5_000_000, 35_000_000)


def lane_shifts(n: int) -> List[int]:
    S = -(-n // 32)
    return [n - min(n, (lane + 1) * S) for lane in range(32)]


def crc_shift_levels() -> Corpus:
    c = Corpus("crc32")
    bits = 0
    for i, n in enumerate(SHIFT_N):
        body = plain_text(n, seed=100 + i)
        for sh in lane_shifts(n):
            bits |= sh
        c.add(framed(body), ref_crc32(body.decode()))
    assert bits & ((1 << SHIFT_BITS) - 1) == (1 << SHIFT_BITS) - 1, bin(bits)
    # multi-MiB bodies with escapes and raw UTF-8 throughout: decoded and raw byte counts differ at the high levels
    rng = np.random.default_rng(5)
    pool = ["a", "q", "7", " ", "é", "€", "\U0001F600", '"', "\\", "\n", "/", " "]
    chunk = "".join(rng.choice(pool, size=1 << 18))
    for reps, ascii_only in ((24, False), (24, True), (96, False)):
        s = "".join(chunk + str(r) for r in range(reps))
        body = json.dumps(s, ensure_ascii=ascii_only)[1:-1].encode()
        c.add(framed(body), ref_crc32(s))
    assert max(len(p) for p in c.payloads) < 64 << 20
    return c


# ------------------------------------------------------------------ windows of small tasks with a few large ones
LARGE = (2 << 10, 20 << 10, 100 << 10, 1 << 20)
MEDIUM = (300, 600, 900, 1500, 3000, 6000)          # runs of these make tiles that overflow while each task still fits


def _string_task(handler: str, size: int, kind: str, rng) -> Tuple[bytes, Want]:
    n = max(1, size - len(FRAME_PRE) - len(FRAME_SUF))
    if kind == "clean":
        body = plain_text(n, seed=int(rng.integers(1 << 30)))
    else:
        pool = ["a", "b", "c", "d", " ", '"', "\\", "\n", "é", "€", "\U0001F600", "/"]
        s = "".join(rng.choice(pool, size=max(1, n // 3)))
        body = json.dumps(s)[1:-1].encode()
        if kind == "upper":                                  # json.dumps's own text with its escapes in upper-case hex
            body = body.replace(b"\\u00e9", b"\\u00E9").replace(b"\\u20ac", b"\\u20AC")
    return framed(body), ref_string(handler, body)


def _vadd(size: int, rng, floats: Optional[int] = None) -> Tuple[bytes, Want]:
    f = floats or max(1, (size - 28) * 3 // 32)
    a = rng.uniform(-1e3, 1e3, size=f).astype(np.float32)
    b = rng.uniform(-1e3, 1e3, size=f).astype(np.float32)
    return vadd_task(a, b)


def _json(size: int, rng, negative: bool = False) -> Tuple[bytes, Want]:
    k = max(1, (size - 60) // 8)
    lo = -10**6 if negative else 0
    vals = rng.integers(lo, 10**6, size=k).tolist()
    p, _ = json_sum_task(vals)
    pad = max(0, size - len(p))
    return json_sum_task(vals, pad=pad, ident=int(rng.integers(1000)))


def handler_task(handler: str, size: int, rng, kind: str = "clean") -> Tuple[bytes, Want]:
    if handler in ("identity", "crc32"):
        return _string_task(handler, size, kind, rng)
    if handler == "vadd_f32":
        return _vadd(size, rng)
    return _json(size, rng, negative=kind == "negative")


def _kinds(handler: str):
    return {"identity": ("clean", "escaped", "upper"), "crc32": ("clean", "escaped"),
            "vadd_f32": ("clean",), "json_sum": ("clean", "negative")}[handler]


def mixed_windows(handler: str, seed: int = 0, n_small: int = 20000) -> Corpus:
    """Mostly small tasks (they keep the stage buffer small), runs of medium ones, and a few of about 2 KiB, 20 KiB,
    100 KiB and 1 MiB. vadd_f32 adds vectors of 4096 and 20 000 floats; json_sum's documents of 1-4 KiB use the
    warp-parallel parser when staged and the sequential one when not."""
    rng = np.random.default_rng(1000 + seed)
    kinds = _kinds(handler)
    items: List[Tuple[bytes, Want]] = []
    for i in range(n_small):
        items.append(handler_task(handler, int(rng.integers(40, 160)), rng, kinds[i % len(kinds)]))
    extra: List[List[Tuple[bytes, Want]]] = []
    for size in MEDIUM:
        for kind in kinds:
            extra.append([handler_task(handler, size + int(rng.integers(0, 64)), rng, kind) for _ in range(6)])
    for size in LARGE:
        for kind in kinds:
            extra.append([handler_task(handler, size, rng, kind)])
    if handler == "vadd_f32":
        extra += [[_vadd(0, rng, floats=4096)], [_vadd(0, rng, floats=20000)], [_vadd(0, rng, floats=4096)] * 2]
    if handler == "json_sum":
        for size in (1100, 2000, 3000, 4000):
            extra.append([_json(size, rng) for _ in range(3)])
    # runs land at random places among the small tasks
    cuts = np.sort(rng.choice(np.arange(1, n_small), size=len(extra), replace=False))
    out, prev = [], 0
    for cut, run in zip(cuts.tolist(), extra):
        out += items[prev:cut] + run
        prev = cut
    out += items[prev:]
    c = Corpus(handler)
    for p, w in out:
        c.add(p, w)
    return c


# ------------------------------------------------------------------ tiles of exactly the stage buffer's size
@dataclass
class FitWindow:
    corpus: Corpus
    pushes: List[int]          # tasks per push (one drain takes the whole window)
    target: int                # the tile's aligned span (contiguous) or sum of aligned spans (scattered)
    scattered: bool


def _sized(handler: str, size: int, rng) -> Tuple[bytes, Want]:
    if handler in ("identity", "crc32"):
        body = plain_text(size - len(FRAME_PRE) - len(FRAME_SUF), seed=int(rng.integers(1 << 30)))
        return framed(body), ref_string(handler, body)
    vals = rng.integers(0, 1000, size=4).tolist()
    p, _ = json_sum_task(vals)
    p, w = json_sum_task(vals, pad=size - len(p))
    assert len(p) == size
    return p, w


VADD_LENS = {f: len(vadd_task(np.zeros(f, np.float32), np.zeros(f, np.float32))[0]) for f in range(1, 64)}


def exact_fit_tiles(handler: str, in_cap: int = 1024) -> List[FitWindow]:
    """One-tile windows (pushed into an empty ring, so the tile starts 16-aligned at ring offset 0) whose aligned span is
    in_cap - 16, in_cap and in_cap + 16; and two-push windows whose scattered tile's aligned spans add up to the same
    three sizes (every task a multiple of 16 bytes, the first push's bytes not a multiple of 256: the second push starts
    at the next 256-byte boundary, so the tile is not contiguous). vadd_f32's payloads are never a multiple of 16 bytes
    long: it gets the contiguous windows only."""
    rng = np.random.default_rng(77)
    out = []
    T = tile_tasks(handler, 1)
    for target in (in_cap - 16, in_cap, in_cap + 16):
        c = Corpus(handler)
        if handler == "vadd_f32":
            # a DP over the payload lengths vadd_f32 can have: r <= T tasks adding up to target
            best = {0: []}
            for _ in range(T):
                nxt = dict(best)
                for tot, fs in best.items():
                    for f, ln in VADD_LENS.items():
                        if tot + ln <= target and tot + ln not in nxt:
                            nxt[tot + ln] = fs + [f]
                best = nxt
            for f in best[target]:
                a = rng.uniform(-1, 1, size=f).astype(np.float32)
                p, w = vadd_task(a, a[::-1].copy())
                c.add(p, w)
        else:
            r = min(T, 4)
            sizes = [target // r] * r
            sizes[-1] += target - sum(sizes)
            for s in sizes:
                c.add(*_sized(handler, s, rng))
        assert sum(len(p) for p in c.payloads) == target and c.n <= T
        out.append(FitWindow(c, [c.n], target, False))
        if handler == "vadd_f32":
            continue
        # scattered: 3 tasks then 1 (T = 4) or 2 + 2 (identity: T = 32), lengths multiples of 16
        c = Corpus(handler)
        units = target // 16
        sizes = [16 * (units // 4 - 1)] * 3
        sizes.append(target - sum(sizes))
        assert all(s % 16 == 0 and s >= 64 for s in sizes)
        first = 3 if sum(sizes[:3]) % 256 else 2
        assert sum(sizes[:first]) % 256
        for s in sizes:
            c.add(*_sized(handler, s, rng))
        out.append(FitWindow(c, [first, 4 - first], target, True))
    return out
