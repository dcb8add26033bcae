"""Keys that collide in the library's GPU hash tables, built from the tables' own home functions.

None of the hashes is seeded, so the keys that share a home slot, wrap from a table's last slot to slot 0, or stay in
one dictionary bucket through growth can be computed exactly.  Every home function is restated here in numpy, with the
source line it was taken from; `SOURCES` lists the constants each restatement depends on, and the CPU tests check that
they still appear in those files (a changed hash makes that test fail instead of letting the GPU tests quietly stop
colliding).

  table                                     home                                                   source
  bucketed key dictionary (window, updating) bucket = mulhi32(bd_hash(k) >> 32, n_buckets)          bdict.cuh bd_bucket
                                            slot = top 11 bits of k * BD_SLOT_MULT, groups of 4    bdict.cuh bd_slot0
  two-pass ingest, pass-2 lookup table      group = top 9 bits of the same product, x 8            ingest_two_pass.cuh
                                            tag = bits 36..43 of the product (0 becomes 1)         p2_group / p2_tag
  session key dictionary                    mulhi32(mix64(k) >> 32, cap)                           dict.cuh dict_home
  instant-window groups                     mix64(mix64(instant) ^ k) & mask                       instant_agg.cu
  instant join build table                  mix64(k ^ mix64(ts)) & mask                            join.cu pair_hash
  join-with-expiration multimap             (mix64(k) >> 20) & mask                                ttl_join.cu tj_home
  shuffle routing                           (mix64(k) / (U64_MAX / n)) % n                         shuffle.cu dest_of
"""
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "arroyo_b200", "csrc")
M64 = (1 << 64) - 1
U64 = np.uint64

# common.cuh mix64: the splitmix64 finaliser
MIX_ADD, MIX_M1, MIX_M2 = 0x9E3779B97F4A7C15, 0xBF58476D1CE4E5B9, 0x94D049BB133111EB
MIX_S = (30, 27, 31)
# bdict.cuh
BD_MULT = 0x9E3779B97F4A7C15       # bd_hash
BD_SLOT_MULT = 0xD6E8FEB86659FD93  # bd_slot0, and p2_hash in ingest_two_pass.cuh
BD_KS, BD_KS_LOG2, BD_GROUP, BD_CAPB, BD_MEAN = 2048, 11, 4, 1280, 1024
# ingest_two_pass.cuh
P2_HS, P2_HG = 4096, 8
# ttl_join.cu tj_home
TJ_SHIFT = 20

# (file, text) pairs every restatement above depends on: each text must appear in the file verbatim
SOURCES = [
    ("common.cuh", "uint64_t z = x + 0x9E3779B97F4A7C15ull;"),
    ("common.cuh", "z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;"),
    ("common.cuh", "z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;"),
    ("common.cuh", "return z ^ (z >> 31);"),
    ("bdict.cuh", "return (k ^ (k >> 32)) * 0x9E3779B97F4A7C15ull;"),
    ("bdict.cuh", "return (uint32_t)(((h >> 32) * (uint64_t)n_buckets) >> 32);"),
    ("bdict.cuh", "(((uint64_t)key * 0xD6E8FEB86659FD93ull) >> (64 - BD_KS_LOG2)) & ~(uint32_t)(BD_GROUP - 1)"),
    ("bdict.cuh", "constexpr int BD_KS = 2048;"),
    ("bdict.cuh", "constexpr int BD_CAPB = 1280;"),
    ("bdict.cuh", "constexpr int BD_MEAN = 1024;"),
    ("bdict.cuh", "constexpr int BD_KS_LOG2 = 11;"),
    ("bdict.cuh", "constexpr int BD_GROUP = 4;"),
    ("ingest_two_pass.cuh", "return (uint32_t)(((uint64_t)key * 0xD6E8FEB86659FD93ull) >> 32);"),
    ("ingest_two_pass.cuh", "return (h >> 23) * P2_HG;"),
    ("ingest_two_pass.cuh", "const uint32_t t = (h >> 4) & 0xFFu;"),
    ("ingest_two_pass.cuh", "constexpr int P2_HS = 4096;"),
    ("ingest_two_pass.cuh", "constexpr int P2_HG = 8;"),
    ("dict.cuh", "return (uint32_t)(((mix64(key) >> 32) * (uint64_t)cap) >> 32);"),
    ("dict.cuh", "return pos + 1 == cap ? 0u : pos + 1;"),
    ("instant_agg.cu", "return (uint32_t)mix64(mix64((uint64_t)inst) ^ (uint64_t)key) & mask;"),
    ("join.cu", "return mix64((uint64_t)key ^ mix64((uint64_t)ts));"),
    ("join.cu", "uint32_t pos = (uint32_t)pair_hash(k, t) & mask;"),
    ("ttl_join.cu", "return (uint32_t)(mix64((uint64_t)key) >> 20) & mask;"),
    ("shuffle.cu", "return (uint32_t)((mix64((uint64_t)key) / range) % n_dest);"),
]


def _u(x):
    return np.asarray(x).astype(np.int64, copy=False).view(np.uint64) if np.asarray(x).dtype != np.uint64 else \
        np.asarray(x, dtype=np.uint64)


def _i64(u):
    return np.asarray(u, dtype=np.uint64).view(np.int64)


# ---- mix64 and its inverse ------------------------------------------------------------------------------------------
def mix64(x):
    """common.cuh mix64 over a uint64 / int64 array (returns uint64)."""
    z = _u(x) + U64(MIX_ADD)
    with np.errstate(over="ignore"):
        z = (z ^ (z >> U64(30))) * U64(MIX_M1)
        z = (z ^ (z >> U64(27))) * U64(MIX_M2)
    return z ^ (z >> U64(31))


def _unshift(y, s):
    """The x with x ^ (x >> s) == y."""
    x = y.copy()
    for _ in range(64 // s + 1):
        x = y ^ (x >> U64(s))
    return x


def mix64_inv(h):
    """The inverse of mix64: every uint64 has exactly one preimage (returns uint64)."""
    z = _unshift(np.asarray(h, dtype=np.uint64), 31)
    with np.errstate(over="ignore"):
        z = _unshift(z * U64(pow(MIX_M2, -1, 1 << 64)), 27)
        z = _unshift(z * U64(pow(MIX_M1, -1, 1 << 64)), 30)
        return z - U64(MIX_ADD)


# ---- home functions -------------------------------------------------------------------------------------------------
def bd_hash(k):
    k = _u(k)
    with np.errstate(over="ignore"):
        return (k ^ (k >> U64(32))) * U64(BD_MULT)


def bd_bucket(k, n_buckets):
    return (((bd_hash(k) >> U64(32)) * U64(n_buckets)) >> U64(32)).astype(np.int64)


def slot_product(k):
    with np.errstate(over="ignore"):
        return _u(k) * U64(BD_SLOT_MULT)


def bd_slot0(k):
    return ((slot_product(k) >> U64(64 - BD_KS_LOG2)).astype(np.int64)) & ~(BD_GROUP - 1)


def p2_group(k):
    return ((slot_product(k) >> U64(32 + 23)).astype(np.int64)) * P2_HG


def p2_tag(k):
    t = ((slot_product(k) >> U64(32 + 4)) & U64(0xFF)).astype(np.int64)
    return np.where(t == 0, 1, t)


def dict_home(k, cap):
    return (((mix64(k) >> U64(32)) * U64(cap)) >> U64(32)).astype(np.int64)


def instant_home(inst, k, mask):
    return (mix64(mix64(inst) ^ _u(k)) & U64(mask)).astype(np.int64)


def pair_home(k, ts, mask):
    return (mix64(_u(k) ^ mix64(ts)) & U64(mask)).astype(np.int64)


def tj_home(k, mask):
    return ((mix64(k) >> U64(TJ_SHIFT)) & U64(mask)).astype(np.int64)


def dest(k, n):
    """shuffle.cu dest_of: (mix64(k) / (U64_MAX / n)) % n."""
    return ((mix64(k) // U64(M64 // n)) % U64(n)).astype(np.int64)


# ---- constructors ---------------------------------------------------------------------------------------------------
def _distinct(keys, n, what):
    keys = np.asarray(keys, dtype=np.int64)
    _, first = np.unique(keys, return_index=True)
    keys = keys[np.sort(first)]
    assert len(keys) >= n, (what, len(keys), n)
    return keys[:n]


def bucketed_chain(n, seed=0, tag="one", split_at=None, max_buckets=4096):
    """`n` keys whose bucketed-dictionary home is the last group of the bucket (slot 2044) and whose pass-2 home is
    the last group of the lookup table (4088), so both chains wrap; with `tag` "one" they share one pass-2 tag, with
    "distinct" their tags run through 1..255.  Without `split_at` they sit in the last bucket at every bucket count up
    to `max_buckets` (no growth splits them).  With `split_at = b`, they share the last bucket at b buckets and split
    evenly between the last two buckets at 2b, so the first doubling rehashes a long chain into two."""
    rng = np.random.default_rng(seed)
    inv = U64(pow(BD_SLOT_MULT, -1, 1 << 64))
    out, need = [], n
    while need > 0:
        free = rng.integers(0, 1 << 63, 1 << 22, dtype=np.uint64) | (rng.integers(0, 2, 1 << 22, dtype=np.uint64) << U64(63))
        p = free | U64(((1 << 11) - 1) << 53)  # top 11 bits: home group 2044 of 2048, pass-2 group 511 of 512
        tags = np.full(len(p), 0xA5, dtype=np.uint64) if tag == "one" else \
            (np.arange(len(p), dtype=np.uint64) % U64(255)) + U64(1)
        p = (p & ~U64(0xFF << 36)) | (tags << U64(36))
        with np.errstate(over="ignore"):
            k = p * inv
        hi = bd_hash(k) >> U64(32)
        if split_at is None:
            lim = max_buckets
            while lim & (lim - 1):
                lim += 1
            keep = hi >= U64((1 << 32) - (1 << 32) // lim)  # last bucket for every count <= lim
        else:
            keep = bd_bucket(k, split_at) == split_at - 1
        k = k[keep]
        if split_at is not None:  # balance the halves at 2b
            lo = k[bd_bucket(k, 2 * split_at) == 2 * split_at - 2]
            up = k[bd_bucket(k, 2 * split_at) == 2 * split_at - 1]
            m = min(len(lo), len(up))
            k = np.stack([lo[:m], up[:m]], 1).reshape(-1)
        out.append(_i64(k))
        need -= len(k)
    return _distinct(np.concatenate(out), n, "bucketed_chain")


def session_chain(n, seed=0):
    """`n` keys with mix64(k) >> 32 == 0xFFFFFFFF: the session dictionary's home is its last slot (cap - 1) at every
    capacity, so every chain wraps."""
    rng = np.random.default_rng(seed)
    low = rng.choice(1 << 32, n, replace=False).astype(np.uint64)
    return _i64(mix64_inv(U64(0xFFFFFFFF << 32) | low))


def ttl_chain(n, seed=0):
    """`n` keys with bits 20..51 of mix64(k) all ones: the multimap's home is its last slot at every mask up to 2^32."""
    rng = np.random.default_rng(seed)
    low = rng.choice(1 << 20, n, replace=False).astype(np.uint64)
    high = rng.integers(0, 1 << 12, n, dtype=np.uint64) << U64(52)
    return _i64(mix64_inv(high | U64(0xFFFFFFFF << 20) | low))


def instant_chain(times, n_per, seed=0):
    """For each timestamp t in `times`, `n_per` keys k with mix64(mix64(t) ^ k) low 32 bits all ones: every (t, k)
    group of the instant window shares the last slot at every mask, across instants.  Returns (ts, keys) arrays."""
    rng = np.random.default_rng(seed)
    times = np.asarray(times, dtype=np.int64)
    ts = np.repeat(times, n_per)
    high = rng.choice(1 << 32, len(ts), replace=False).astype(np.uint64) << U64(32)
    k = mix64_inv(high | U64(0xFFFFFFFF)) ^ mix64(ts)
    return ts, _i64(k)


# the instant join's pair hash, mix64(k ^ mix64(ts)), has the instant window's form: the same keys collide in both
pair_chain = instant_chain


def routed(n, where, seed=0):
    """`n` keys that every n_dest in (2, 3, 8) routes to destination 0 (`where` = "first") or n_dest - 1 ("last")."""
    rng = np.random.default_rng(seed)
    low = rng.choice(1 << 39, n, replace=False).astype(np.uint64)
    h = low if where == "first" else U64(M64 - (1 << 40)) - low
    return _i64(mix64_inv(h))


ORIGIN = 1_700_000_000 * 1_000_000_000


def families(n_per=300):
    """Structured key families a real stream has: j << s, ORIGIN + j * 10^9, and keys whose halves are equal."""
    j = np.arange(1, n_per + 1, dtype=np.uint64)
    fams = {}
    for s in (0, 8, 16, 32, 48, 53, 56, 60):
        m = min(n_per, (1 << (64 - s)) - 1)  # j << 60 has 15 distinct nonzero values
        fams[f"shift{s}"] = _i64(j[:m] << U64(s))
    fams["origin_ns"] = ORIGIN + np.arange(n_per, dtype=np.int64) * 1_000_000_000
    fams["halves"] = _i64(j | (j << U64(32)))
    return fams
