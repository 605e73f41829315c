"""Host-side logic of the multi-GPU path: how the virtual nodes are split across ranks and what the sharded tally
protocol computes.  Pure Python/numpy so that it can be exercised with `gloo` on CPU; the GPU library implements the same
protocol in csrc/fast_paxos.cu (rapid_fp_tally_cd with a communicator)."""
import numpy as np

HIST_BUCKETS = 1 << 16


def shard_range(n, rank, world):
    """contiguous slice of ring-0 positions owned by `rank` ("nodes shard by ring hash")"""
    begin = rank * n // world
    return begin, (rank + 1) * n // world - begin


def histogram_of(h1, counts=None):
    """65 536-bucket histogram over the top 16 bits of the proposal fingerprints voted on this rank"""
    h1 = np.asarray(h1, np.uint64)
    w = np.ones(len(h1), np.int64) if counts is None else np.asarray(counts, np.int64)
    return np.bincount((h1 >> np.uint64(48)).astype(np.int64), weights=w, minlength=HIST_BUCKETS).astype(np.int32)


def verification_words(h1, h2, ln, bucket):
    """(max h1, max ~h1, max h2, max ~h2, max len, max ~len) over this rank's entries in `bucket`; zeros if none"""
    h1 = np.asarray(h1, np.uint64); h2 = np.asarray(h2, np.uint64); ln = np.asarray(ln, np.uint64)
    m = (h1 >> np.uint64(48)).astype(np.int64) == bucket
    if not m.any():
        return np.zeros(6, np.uint64)
    return np.array([h1[m].max(), (~h1[m]).max(), h2[m].max(), (~h2[m]).max(), ln[m].max(), (~ln[m]).max()], np.uint64)


def decide(global_hist, global_words_of, quorum):
    """the decision every rank reaches after the sum all-reduce (global_hist) and the max all-reduce of the winning
    bucket's verification words (global_words_of(bucket)).  Returns (decided, h1, h2, len, count)."""
    cand = np.nonzero(global_hist >= quorum)[0]
    if len(cand) == 0:
        return False, 0, 0, 0, 0
    b = int(cand[0])
    w = global_words_of(b)
    single = w[0] == ~w[1] and w[2] == ~w[3] and w[4] == ~w[5]
    if not single:
        return False, 0, 0, 0, 0          # two proposals share the bucket: the library refines digit by digit
    return True, int(w[0]), int(w[2]), int(w[4]), int(global_hist[b])


# ---- the single-all-reduce protocol (csrc/fast_paxos.cu: phase S of k_fp_tally / k_fp_decide_sum) ------------------
SUM_BUCKETS, SUM_WORDS = 4096, 8
_M64 = (1 << 64) - 1


def _splitmix64(x):
    x = (x + 0x9E3779B97F4A7C15) & _M64
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & _M64
    return x ^ (x >> 31)


def _check_word(h1, h2, ln):
    rot = ((h2 << 17) | (h2 >> 47)) & _M64
    return _splitmix64(h1 ^ rot ^ ((ln * 0x9E3779B97F4A7C15) & _M64))


def sum_buffer_of(h1, h2, ln, votes_received):
    """this rank's contribution: per 12-bit bucket, count-weighted sums of (1, h1 hi/lo, h2 hi/lo, len, check hi/lo);
    the last row carries votesReceived.  uint64 arithmetic wraps like the device's."""
    buf = [0] * ((SUM_BUCKETS + 1) * SUM_WORDS)
    for a, b, l in zip(h1, h2, ln):
        a, b, l = int(a), int(b), int(l)
        m = _check_word(a, b, l)
        o = (a >> 52) * SUM_WORDS
        for k, v in enumerate((1, a >> 32, a & 0xFFFFFFFF, b >> 32, b & 0xFFFFFFFF, l, m >> 32, m & 0xFFFFFFFF)):
            buf[o + k] = (buf[o + k] + v) & _M64
    buf[SUM_BUCKETS * SUM_WORDS] = int(votes_received)
    return np.array(buf, dtype=np.uint64)


def decide_sum(global_buf, quorum):
    """what every rank concludes from the summed buffer: (decided, h1, h2, len, count, votes_received, ambiguous)"""
    g = [int(x) for x in global_buf]
    received = g[SUM_BUCKETS * SUM_WORDS]
    for b in range(SUM_BUCKETS):
        w = g[b * SUM_WORDS: (b + 1) * SUM_WORDS]
        c = w[0]
        if c < quorum or c == 0:
            continue
        if any(x % c for x in w[1:]):
            return False, 0, 0, 0, 0, received, True
        a1, a2, b1, b2, ln = (w[k] // c for k in range(1, 6))
        if max(a1, a2, b1, b2) > 0xFFFFFFFF:
            return False, 0, 0, 0, 0, received, True
        h1, h2 = (a1 << 32) | a2, (b1 << 32) | b2
        m = _check_word(h1, h2, ln)
        if w[6] // c != m >> 32 or w[7] // c != m & 0xFFFFFFFF or (h1 >> 52) != b:
            return False, 0, 0, 0, 0, received, True
        return True, h1, h2, ln, c, received, False
    return False, 0, 0, 0, 0, received, False
