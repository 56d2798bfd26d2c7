"""numpy-vectorised restatement of NTL's seeded stream and of DoubleCRT::randomize (TEST INFRASTRUCTURE, part of the oracle).

The same bytes and the same consumption pattern as ntl_prg.RandomStream + pyoracle.randomize_rows (tests check the two
against each other), fast enough for full-size key-switching matrices: one config-3 matrix is 3 x 35 rows of 2^16
residues, about 60 MB of key stream.

DoubleCRT::randomize (src/DoubleCRT.cpp:1258-1378) only ever takes whole 2048-byte buffers from the stream, and the stream
starts at block 0 after SetSeed, so buffer b is exactly the ChaCha20 blocks 32b .. 32b+31: BufferStream hands out
buffers by index.
"""
import numpy as np

import ntl_prg

BUF = 2048


def seed_key(seed) -> bytes:
    """The ChaCha20 key of NTL::SetSeed for a non-negative int seed, or for its little-endian magnitude bytes
    (high-order zero bytes do not count, as NumBytes ignores them)."""
    data = ntl_prg.zz_bytes(seed) if isinstance(seed, int) else bytes(seed).rstrip(b"\0")
    return ntl_prg.derive_key(data)


def chacha20_blocks(key: bytes, first: int, count: int) -> np.ndarray:
    """Key-stream blocks first .. first+count-1 as count*64 uint8 (the bytes of ntl_prg.chacha20_block)."""
    k = np.frombuffer(key, dtype="<u4")
    ctr = np.arange(first, first + count, dtype=np.uint64)
    st = [np.full(count, c, dtype=np.uint32) for c in (0x61707865, 0x3320646E, 0x79622D32, 0x6B206574)]
    st += [np.full(count, k[i], dtype=np.uint32) for i in range(8)]
    st += [(ctr & np.uint64(0xFFFFFFFF)).astype(np.uint32), (ctr >> np.uint64(32)).astype(np.uint32),
           np.zeros(count, dtype=np.uint32), np.zeros(count, dtype=np.uint32)]
    x = [s.copy() for s in st]

    def rotl(v, n):
        return (v << np.uint32(n)) | (v >> np.uint32(32 - n))

    def qr(a, b, c, d):
        x[a] += x[b]; x[d] = rotl(x[d] ^ x[a], 16)
        x[c] += x[d]; x[b] = rotl(x[b] ^ x[c], 12)
        x[a] += x[b]; x[d] = rotl(x[d] ^ x[a], 8)
        x[c] += x[d]; x[b] = rotl(x[b] ^ x[c], 7)

    for _ in range(10):
        qr(0, 4, 8, 12); qr(1, 5, 9, 13); qr(2, 6, 10, 14); qr(3, 7, 11, 15)
        qr(0, 5, 10, 15); qr(1, 6, 11, 12); qr(2, 7, 8, 13); qr(3, 4, 9, 14)
    words = np.stack([a + b for a, b in zip(x, st)], axis=1).astype("<u4")   # [count][16]
    return words.view(np.uint8).reshape(-1)


class BufferStream:
    """NTL's RandomStream after SetSeed as DoubleCRT::randomize consumes it: 2048-byte buffers, in order."""

    def __init__(self, seed):
        self.key, self.next = seed_key(seed), 0

    def peek(self, count: int) -> np.ndarray:
        """The next `count` buffers, [count][2048] uint8, not consumed."""
        return chacha20_blocks(self.key, 32 * self.next, 32 * count).reshape(count, BUF)

    def consume(self, count: int):
        self.next += count


def randomize_rows(primes, phim: int, idxs, stream: BufferStream) -> dict:
    """pyoracle.randomize_rows over a BufferStream: {i: uint64[phim]} for i in sorted(idxs).  Per row: fresh buffers,
    nb = ceil(k/8) little-endian bytes per candidate (k = bits(q-1)), masked to k bits, accepted when < q,
    floor(2048/nb) candidates per buffer; the rest of the row's last buffer is discarded."""
    rows = {}
    for i in sorted(idxs):
        q = int(primes[i])
        k = (q - 1).bit_length()
        nb = (k + 7) // 8
        c = BUF // nb
        parts, have = [], 0
        while have < phim:
            step = max(4, int((phim - have) / (c * q / 2 ** k) * 1.05) + 2)
            cand = stream.peek(step)[:, :c * nb].reshape(step, c, nb).astype(np.uint64)
            v = np.zeros((step, c), dtype=np.uint64)
            for b in range(nb):
                v |= cand[:, :, b] << np.uint64(8 * b)
            v &= np.uint64((1 << k) - 1)
            ok = v < np.uint64(q)
            cum = have + np.cumsum(ok.sum(axis=1))
            used = int(np.searchsorted(cum, phim)) + 1 if cum[-1] >= phim else step
            parts.append(v[:used][ok[:used]])
            have = int(cum[used - 1])
            stream.consume(used)
        rows[i] = np.concatenate(parts)[:phim]
    return rows
