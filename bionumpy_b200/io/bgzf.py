"""BGZF output (SAM specification 4.1): a ``.gz`` file of independent gzip members of at most 65280 input bytes each,
every member carrying the 'BC' extra field with its size, closed by the 28-byte empty EOF member.  gzip and zcat read
it as ordinary multi-member gzip; this package's reader inflates its blocks in parallel (ingest._bgzf_blocks).  Blocks
are deflated in parallel on the ingest thread pool (zlib releases the GIL) and written in order."""
import struct
import zlib

BLOCK_INPUT = 65280             # input bytes per block: the deflated block always fits the 16-bit BSIZE
BATCH_BLOCKS = 64               # blocks deflated in parallel per batch (~4 MiB of input)
EOF_BLOCK = bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")


def compress_block(data) -> bytes:
    """One BGZF member: raw deflate at zlib's default level, the BC extra field, CRC32 and ISIZE."""
    c = zlib.compressobj(zlib.Z_DEFAULT_COMPRESSION, zlib.DEFLATED, -15)
    payload = c.compress(data) + c.flush()
    header = struct.pack("<BBBBIBBHBBHH", 0x1F, 0x8B, 8, 4, 0, 0, 0xFF, 6, 66, 67, 2, len(payload) + 25)
    return header + payload + struct.pack("<II", zlib.crc32(data) & 0xFFFFFFFF, len(data))


class BgzfWriter:
    """A write-only file object over ``raw`` (opened "wb" or "ab": appending adds members after the old EOF block,
    which readers skip as an empty member)."""

    def __init__(self, raw):
        self._raw = raw
        self._pending = bytearray()
        self.name = getattr(raw, "name", None)

    def write(self, data):
        self._pending += data
        if len(self._pending) >= BLOCK_INPUT * BATCH_BLOCKS:
            n_full = len(self._pending) // BLOCK_INPUT * BLOCK_INPUT
            self._emit(n_full)
        return len(data)

    def _emit(self, n):
        from .ingest import _pool
        view = bytes(self._pending[:n])
        del self._pending[:n]
        futs = [_pool().submit(compress_block, view[a:a + BLOCK_INPUT]) for a in range(0, n, BLOCK_INPUT)]
        for f in futs:
            self._raw.write(f.result())

    def flush(self):
        if self._pending:
            self._emit(len(self._pending))
        self._raw.flush()

    def close(self):
        if self._raw is None:
            return
        try:
            if self._pending:
                self._emit(len(self._pending))
            self._raw.write(EOF_BLOCK)
        finally:
            self._raw.close()
            self._raw = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()
