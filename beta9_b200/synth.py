"""Deterministic synthetic task batches for BASELINE.json's five configs (SURVEY.md §8d).

Everything is seeded with 0xB9. A batch is the packed form the C ABI takes (include/b9gpu.h):
`task_ids` uint8[n,16], `payload` uint8[total] (the TaskQueuePutRequest.payload bytes of every
task, back to back, exactly as `_CallableWrapper.put` builds them —
sdk/src/beta9/abstractions/taskqueue.py:284-285: `json.dumps({"args": args, "kwargs": kwargs})`)
and `offsets` uint64[n+1].

Input generation only: no oracle code, no device code.
"""
from __future__ import annotations

import base64
import json
from dataclasses import dataclass
from typing import List, Optional

import numpy as np

SEED = 0xB9

# `{"args": ["` ... `"], "kwargs": {}}` — what json.dumps emits around a single string argument
PREFIX = b'{"args": ["'
SUFFIX = b'"], "kwargs": {}}'

# printable ASCII minus the five characters Go's HTML-safe encoder or JSON itself must escape
PLAIN_ALPHABET = np.array([c for c in range(0x20, 0x7F) if chr(c) not in '"\\<>&'], dtype=np.uint8)
# adversarial pool: everything that exercises an escape rule somewhere on the path
ADVERSARIAL_POOL = (
    ['"', "\\", "<", ">", "&", "/", "\n", "\r", "\t", "\b", "\f", "\x01", "\x1f", "\x7f",
     "\u00e9", "\u00df", "\u2028", "\u2029", "\ufffd", "\u20ac", "\U0001f600", "\U00010348",
     "\ud83d", "\udc00"]
    + [chr(c) for c in range(0x20, 0x7F)]
)


@dataclass
class Batch:
    task_ids: np.ndarray      # uint8 [n,16]
    payload: np.ndarray       # uint8 [total]
    offsets: np.ndarray       # uint64 [n+1]
    name: str = ""

    @property
    def n(self) -> int:
        return int(self.offsets.shape[0] - 1)

    def task(self, i: int) -> bytes:
        return self.payload[int(self.offsets[i]):int(self.offsets[i + 1])].tobytes()

    def tasks(self) -> List[bytes]:
        return [self.task(i) for i in range(self.n)]

    def slice(self, lo: int, hi: int) -> "Batch":
        o = self.offsets[lo:hi + 1]
        return Batch(self.task_ids[lo:hi].copy(), self.payload[int(o[0]):int(o[-1])].copy(),
                     (o - o[0]).astype(np.uint64), self.name)


def _splitmix64(x: np.ndarray) -> np.ndarray:
    x = (x + np.uint64(0x9E3779B97F4A7C15)).astype(np.uint64)
    z = x
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def task_ids(n: int, seed: int = SEED, start: int = 0) -> np.ndarray:
    """task i -> 16 bytes = splitmix64 in counter mode over (seed, 2i) and (seed, 2i+1), with the
    RFC 4122 version-4 / variant bits forced so the string form looks like uuid.NewV4()'s
    (pkg/task/dispatch.go:56)."""
    with np.errstate(over="ignore"):
        i = np.arange(start, start + n, dtype=np.uint64)
        base = np.uint64(seed) * np.uint64(0xD1342543DE82EF95)
        hi = _splitmix64(base + np.uint64(2) * i)
        lo = _splitmix64(base + np.uint64(2) * i + np.uint64(1))
    out = np.empty((n, 16), dtype=np.uint8)
    out[:, :8] = hi.view(np.uint8).reshape(n, 8)
    out[:, 8:] = lo.view(np.uint8).reshape(n, 8)
    out[:, 6] = (out[:, 6] & 0x0F) | 0x40
    out[:, 8] = (out[:, 8] & 0x3F) | 0x80
    return out


def _pack(chunks: List[bytes], lens: np.ndarray, ids: np.ndarray, name: str) -> Batch:
    payload = np.frombuffer(b"".join(chunks), dtype=np.uint8).copy()
    offsets = np.zeros(len(lens) + 1, dtype=np.uint64)
    np.cumsum(lens, out=offsets[1:])
    assert int(offsets[-1]) == payload.size
    return Batch(ids, payload, offsets, name)


def strings_batch(n: int, chars: int, adversarial_frac: float = 0.01, seed: int = SEED,
                  name: str = "identity") -> Batch:
    """configs[0] (n=10k, chars=64) and configs[1] (n=1M, chars=256): one string argument of
    `chars` characters; `adversarial_frac` of the tasks draw from ADVERSARIAL_POOL instead of the
    plain alphabet, so their JSON form is longer than chars+27 bytes."""
    rng = np.random.default_rng(seed)
    body = PLAIN_ALPHABET[rng.integers(0, PLAIN_ALPHABET.size, size=(n, chars))]
    rows = np.empty((n, chars + len(PREFIX) + len(SUFFIX)), dtype=np.uint8)
    rows[:, :len(PREFIX)] = np.frombuffer(PREFIX, np.uint8)
    rows[:, len(PREFIX):len(PREFIX) + chars] = body
    rows[:, len(PREFIX) + chars:] = np.frombuffer(SUFFIX, np.uint8)
    n_adv = int(round(n * adversarial_frac))
    adv_idx = np.sort(rng.choice(n, size=n_adv, replace=False)) if n_adv else np.empty(0, np.int64)
    lens = np.full(n, rows.shape[1], dtype=np.uint64)
    chunks: List[bytes] = []
    prev = 0
    pool = ADVERSARIAL_POOL
    for k, i in enumerate(adv_idx):
        i = int(i)
        if i > prev:
            chunks.append(rows[prev:i].tobytes())
        picks = rng.integers(0, len(pool), size=chars)
        s = "".join(pool[int(j)] for j in picks)
        b = json.dumps({"args": (s,), "kwargs": {}}).encode("utf-8")
        chunks.append(b)
        lens[i] = len(b)
        prev = i + 1
    if prev < n:
        chunks.append(rows[prev:].tobytes())
    return _pack(chunks, lens, task_ids(n, seed), name)


def zipf_lengths(n: int, seed: int = SEED) -> np.ndarray:
    """configs[2]: 32 + min(4064, zipf(a=1.2) - 1), i.e. clipped to [32, 4096]."""
    rng = np.random.default_rng(seed + 1)
    z = rng.zipf(1.2, size=n).astype(np.int64)
    return (32 + np.minimum(4064, z - 1)).astype(np.int64)


def crc_batch(n: int, seed: int = SEED, lengths: Optional[np.ndarray] = None, name: str = "crc32",
              chunk_tasks: int = 65536) -> Batch:
    """configs[2]: one string argument of zipf length, characters uniform over 0x20..0x7E
    (so `"` and `\\` occur and json.dumps escapes them). Built in chunks to bound memory."""
    rng = np.random.default_rng(seed + 2)
    L = zipf_lengths(n, seed) if lengths is None else np.asarray(lengths, dtype=np.int64)
    joint = np.frombuffer(SUFFIX + PREFIX, np.uint8)
    parts: List[np.ndarray] = []
    lens = np.empty(n, dtype=np.uint64)
    for lo in range(0, n, chunk_tasks):
        hi = min(n, lo + chunk_tasks)
        Lc = L[lo:hi]
        total_chars = int(Lc.sum())
        chars = rng.integers(0x20, 0x7F, size=total_chars, dtype=np.uint8)
        esc = (chars == 0x22) | (chars == 0x5C)
        # json.dumps writes '"' and '\\' as two bytes: insert a backslash before each
        body = np.insert(chars, np.flatnonzero(esc), 0x5C)
        cw = np.zeros(total_chars + 1, dtype=np.int64)
        np.cumsum(esc, out=cw[1:])
        char_off = np.zeros(hi - lo + 1, dtype=np.int64)
        np.cumsum(Lc, out=char_off[1:])
        body_off = char_off + cw[char_off]            # task boundaries inside `body`
        lens[lo:hi] = (np.diff(body_off) + len(PREFIX) + len(SUFFIX)).astype(np.uint64)
        inner = body_off[1:-1]
        framed = np.insert(body, np.repeat(inner, joint.size), np.tile(joint, inner.size))
        parts.append(np.frombuffer(PREFIX, np.uint8))
        parts.append(framed)
        parts.append(np.frombuffer(SUFFIX, np.uint8))
    payload = np.concatenate(parts) if parts else np.empty(0, np.uint8)
    offsets = np.zeros(n + 1, dtype=np.uint64)
    np.cumsum(lens, out=offsets[1:])
    assert int(offsets[-1]) == payload.size
    return Batch(task_ids(n, seed), payload, offsets, name)


def vadd_batch(n: int, floats_per_vec: int = 32, seed: int = SEED, name: str = "vadd_f32") -> Batch:
    """configs[3]: 256 B = 64 little-endian fp32 (a||b), uniform [-1,1), carried as one
    std-base64 string argument (344 characters)."""
    rng = np.random.default_rng(seed + 3)
    v = rng.uniform(-1.0, 1.0, size=(n, 2 * floats_per_vec)).astype("<f4")
    raw = v.view(np.uint8).reshape(n, -1)
    b64 = _b64_rows(raw)
    rows = np.empty((n, b64.shape[1] + len(PREFIX) + len(SUFFIX)), dtype=np.uint8)
    rows[:, :len(PREFIX)] = np.frombuffer(PREFIX, np.uint8)
    rows[:, len(PREFIX):len(PREFIX) + b64.shape[1]] = b64
    rows[:, len(PREFIX) + b64.shape[1]:] = np.frombuffer(SUFFIX, np.uint8)
    lens = np.full(n, rows.shape[1], dtype=np.uint64)
    offsets = np.zeros(n + 1, dtype=np.uint64)
    np.cumsum(lens, out=offsets[1:])
    return Batch(task_ids(n, seed), rows.reshape(-1), offsets, name)


def vadd_special_batch(n: int, floats_per_vec: int = 32, seed: int = SEED, name: str = "vadd_f32_special") -> Batch:
    """vadd_f32 payloads over raw random bit patterns (NaNs with payloads, infinities, denormals,
    signed zeros, overflow to inf): the cases where an fp32 add is more than rounding."""
    rng = np.random.default_rng(seed + 33)
    bits = rng.integers(0, 1 << 32, size=(n, 2 * floats_per_vec), dtype=np.uint64).astype(np.uint32)
    special = np.array([0x7F800000, 0xFF800000, 0x7FC00000, 0xFFC00000, 0x7FA00001, 0xFFA12345, 0x00000001, 0x80000001,
                        0x007FFFFF, 0x00000000, 0x80000000, 0x7F7FFFFF, 0xFF7FFFFF, 0x3F800000, 0xBF800000, 0x7FFFFFFF], np.uint32)
    pick = rng.random(bits.shape) < 0.5
    bits[pick] = special[rng.integers(0, special.size, size=int(pick.sum()))]
    raw = bits.view(np.uint8).reshape(n, -1)
    b64 = _b64_rows(raw)
    rows = np.empty((n, b64.shape[1] + len(PREFIX) + len(SUFFIX)), dtype=np.uint8)
    rows[:, :len(PREFIX)] = np.frombuffer(PREFIX, np.uint8)
    rows[:, len(PREFIX):len(PREFIX) + b64.shape[1]] = b64
    rows[:, len(PREFIX) + b64.shape[1]:] = np.frombuffer(SUFFIX, np.uint8)
    offsets = np.arange(n + 1, dtype=np.uint64) * np.uint64(rows.shape[1])
    return Batch(task_ids(n, seed), rows.reshape(-1), offsets, name)


_B64 = np.frombuffer(b"ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789+/", np.uint8)


def _b64_rows(raw: np.ndarray) -> np.ndarray:
    """std-base64 of every row of a uint8 [n, m] array (vectorised)."""
    n, m = raw.shape
    pad = (-m) % 3
    r = np.concatenate([raw, np.zeros((n, pad), np.uint8)], axis=1).reshape(n, -1, 3).astype(np.uint32)
    w = (r[:, :, 0] << 16) | (r[:, :, 1] << 8) | r[:, :, 2]
    out = np.empty((n, w.shape[1], 4), dtype=np.uint8)
    out[:, :, 0] = _B64[(w >> 18) & 63]
    out[:, :, 1] = _B64[(w >> 12) & 63]
    out[:, :, 2] = _B64[(w >> 6) & 63]
    out[:, :, 3] = _B64[w & 63]
    out = out.reshape(n, -1)
    if pad:
        out[:, -pad:] = ord("=")
    assert out[0].tobytes() == base64.b64encode(raw[0].tobytes())
    return out


def json_batch(n: int, doc_bytes: int = 1024, seed: int = SEED, name: str = "json_sum") -> Batch:
    """configs[4]: one dict argument `{"id": i, "values": [ints in [0,1e6)], "pad": "xxx"}` whose
    JSON text is exactly `doc_bytes` long (the "pad" string tops it up)."""
    rng = np.random.default_rng(seed + 4)
    chunks: List[bytes] = []
    lens = np.empty(n, dtype=np.uint64)
    for i in range(n):
        k = int(rng.integers(60, 120))
        vals = rng.integers(0, 10**6, size=k).tolist()
        doc = {"id": i, "values": vals, "pad": ""}
        cur = len(json.dumps(doc))
        while cur > doc_bytes:
            vals.pop()
            cur = len(json.dumps(doc))
        doc["pad"] = "x" * (doc_bytes - cur)
        b = json.dumps({"args": (doc,), "kwargs": {}}).encode("utf-8")
        chunks.append(b)
        lens[i] = len(b)
    return _pack(chunks, lens, task_ids(n, seed), name)


def _float_value(rng: np.random.Generator):
    """One number of json_float_batch: short decimals, 17-digit values, subnormals, values >= 1e21, integers above 2^53,
    small integers."""
    k = int(rng.integers(0, 8))
    if k == 0:
        return round(float(rng.uniform(-1000, 1000)), int(rng.integers(0, 4)))     # 12.5, -0.37, 401.0
    if k == 1:
        return float(rng.uniform(-1, 1)) * 10.0 ** int(rng.integers(-8, 9))          # 16-17 digits
    if k == 2:
        return float(np.uint64(rng.integers(1, 1 << 52)).view(np.float64)) * (1 if rng.random() < 0.5 else -1)   # subnormal
    if k == 3:
        return float(rng.uniform(1, 10)) * 10.0 ** int(rng.integers(21, 300))       # >= 1e21
    if k == 4:
        return int(rng.integers(1 << 53, 1 << 57)) * (1 if rng.random() < 0.7 else -1)   # above 2^53; sums stay in a C long
    if k == 5:
        return float(rng.integers(-10**6, 10**6))                                  # integral floats: 7.0
    return int(rng.integers(0, 10**6))


def json_float_batch(n: int, doc_bytes: int = 1024, seed: int = SEED, name: str = "json_sum_f64") -> Batch:
    """configs[4]'s document shape `{"id": i, "values": [...], "pad": "xxx"}` with float64 values (see _float_value),
    about `doc_bytes` of JSON text each."""
    rng = np.random.default_rng(seed + 5)
    chunks: List[bytes] = []
    lens = np.empty(n, dtype=np.uint64)
    for i in range(n):
        vals = []
        doc = {"id": i, "values": vals, "pad": ""}
        cur = len(json.dumps(doc))
        while cur < doc_bytes - 40:
            vals.append(_float_value(rng))
            cur += len(json.dumps(vals[-1])) + (2 if len(vals) > 1 else 0)
        doc["pad"] = "x" * max(0, doc_bytes - cur)
        b = json.dumps({"args": (doc,), "kwargs": {}}).encode("utf-8")
        chunks.append(b)
        lens[i] = len(b)
    return _pack(chunks, lens, task_ids(n, seed), name)


_VALUE_STRINGS = ["", "a", "abc", "café", "<tag>", "line\nbreak", "q\"uote", "\U0001f600", " ", "tab\t", "back\\slash", "key"]


def _sdk_value(rng: np.random.Generator, depth: int):
    k = int(rng.integers(0, 10 if depth < 4 else 6))
    if k == 0:
        return bool(rng.random() < 0.5)
    if k == 1:
        return None if rng.random() < 0.3 else int(rng.integers(-10**6, 10**6))
    if k == 2:
        return _float_value(rng)
    if k in (3, 4):
        return _VALUE_STRINGS[int(rng.integers(0, len(_VALUE_STRINGS)))] + str(int(rng.integers(0, 100)))
    if k == 5:
        return round(float(rng.uniform(-100, 100)), int(rng.integers(0, 6)))
    if k in (6, 7):
        return [_sdk_value(rng, depth + 1) for _ in range(int(rng.integers(0, 6)))]
    keys = ["id", "name", "value", "a", "b", "x", "été", "Z", "items", "k" + str(int(rng.integers(0, 9)))]
    return {keys[int(j)]: _sdk_value(rng, depth + 1) for j in rng.integers(0, len(keys), size=int(rng.integers(0, 7)))}


def values_batch(n: int, seed: int = SEED, name: str = "identity_values") -> Batch:
    """SDK payloads `json.dumps({"args": (v,), "kwargs": {}})` of random nested lists and dicts (and some bare numbers)
    holding numbers, strings, booleans and None."""
    rng = np.random.default_rng(seed + 6)
    chunks: List[bytes] = []
    lens = np.empty(n, dtype=np.uint64)
    for i in range(n):
        r = rng.random()
        v = _float_value(rng) if r < 0.1 else ([_sdk_value(rng, 1) for _ in range(int(rng.integers(1, 8)))] if r < 0.55 else
                                                 {"id": i, "data": _sdk_value(rng, 1), "tags": [_sdk_value(rng, 2) for _ in range(3)]})
        b = json.dumps({"args": (v,), "kwargs": {}}).encode("utf-8")
        chunks.append(b)
        lens[i] = len(b)
    return _pack(chunks, lens, task_ids(n, seed), name)


def concat(batches: List[Batch]) -> Batch:
    ids = np.concatenate([b.task_ids for b in batches])
    payload = np.concatenate([b.payload for b in batches])
    lens = np.concatenate([np.diff(b.offsets) for b in batches])
    offsets = np.zeros(lens.size + 1, dtype=np.uint64)
    np.cumsum(lens, out=offsets[1:])
    return Batch(ids, payload, offsets, "+".join(b.name for b in batches))


def from_payloads(payloads: List[bytes], seed: int = SEED, name: str = "custom") -> Batch:
    lens = np.array([len(p) for p in payloads], dtype=np.uint64)
    return _pack(list(payloads), lens, task_ids(len(payloads), seed), name)
