"""Restatement of the reference's bulk write path, for the tests.  TEST INFRASTRUCTURE ONLY.

lib/server/src/db/loading.rs:361-377 update_many_items walks an /update-row body entry by entry and applies each through
update_item (:301-315), which checks the length, reads the big-endian db_idx and calls update_item_raw (:317-359).  Here the
same walk applies the entries in order into a host database in the reference layout [slice][z][ii][j] (one packed word per
item and z), converting each item with the CPU oracle's update_item_raw.  Where the reference panics (a header or chunk that
runs past the end of the body, chunk_len < 4) the walk reports an error, as it does for InvalidLength and a bad db idx; the
entries before the first bad one stay applied.  Nothing here uses the product's parser."""
import numpy as np


def walk_body(body, max_chunk_len, num_items):
    """The loop of update_many_items without the writes: yields (pos, chunk_len, db_idx) per entry that update_item accepts,
    then returns (error message or None, largest_update over the accepted entries)."""
    body = bytes(body)
    offs, largest = 0, 0
    while offs < len(body):
        if offs + 4 > len(body):
            return "header past the end", largest                      # body[offs..offs + 4] panics
        chunk_len = int.from_bytes(body[offs:offs + 4], "big")
        if offs + 4 + chunk_len > len(body):
            return "chunk past the end", largest                       # body[offs + 4..offs + 4 + chunk_len] panics
        if chunk_len > max_chunk_len:
            return "InvalidLength", largest                            # update_item :308-310
        if chunk_len < 4:
            return "chunk shorter than db_idx", largest                # body[..4] panics
        db_idx = int.from_bytes(body[offs + 4:offs + 8], "big")
        if db_idx >= num_items:
            return "bad db idx", largest                               # update_item_raw :333-340
        largest = max(largest, chunk_len)
        yield offs, chunk_len, db_idx
        offs += 4 + chunk_len
    return None, largest


def walk(body, max_chunk_len, num_items):
    """walk_body collected: (entries, error or None, largest_update)."""
    gen = walk_body(body, max_chunk_len, num_items)
    entries = []
    while True:
        try:
            entries.append(next(gen))
        except StopIteration as stop:
            err, largest = stop.value
            return entries, err, largest


def limits(P):
    """(max_chunk_len, num_items) of oracle params P."""
    return 4 + P.slices * P.bytes_per_chunk, P.dim0 * P.num_per


def update_many_items(P, body, db=None):
    """Apply `body` in order to `db` (uint64 [slices][N][num_per][dim0], zeros when None).  Returns
    (db, largest_update, error or None, applied entries [(db_idx, data bytes)])."""
    if db is None:
        db = np.zeros((P.slices, P.N, P.num_per, P.dim0), dtype=np.uint64)
    body = bytes(body)
    entries, err, largest = walk(body, *limits(P))
    applied = []
    for pos, chunk_len, db_idx in entries:
        data = np.frombuffer(body[pos + 8:pos + 4 + chunk_len], dtype=np.uint8)
        db[:, :, db_idx % P.num_per, db_idx // P.num_per] = P.update_item_raw(data).reshape(P.slices, P.N)
        applied.append((db_idx, data))
    return db, largest, err, applied


def read_back(P, db, items, idx, sparse_fold):
    """The bytes ([slices * bytes_per_chunk] uint8) a private read of item `idx` decodes to from `db` (as update_many_items
    returns it), where `items` maps every written db_idx to its bytes.  The dense fold returns item idx.  lib/server's fold
    (compute/fold.rs:37-43) keeps the non-zero ciphertext of a pair when the other is all-zero, whichever one the query
    selects, so in a slice where the target's second-dimension row is empty it can return another row's item of the same
    column."""
    num_per, bpc = P.num_per, P.bytes_per_chunk
    ii, j = idx % num_per, idx // num_per
    nonzero = (db.reshape(P.slices, P.N, num_per, P.dim0) != 0).any(axis=(1, 3))
    out = np.zeros((P.slices, bpc), dtype=np.uint8)
    for s in range(P.slices):
        row = ii
        if sparse_fold:
            cand = [r if nonzero[s, r] else None for r in range(num_per)]
            half, bit = num_per // 2, P.nu_2 - 1           # round k folds rows i and i + half by bit nu_2 - 1 - k of ii
            while half >= 1:
                sel = (ii >> bit) & 1
                for i in range(half):
                    a, b = cand[i], cand[i + half]
                    cand[i] = b if a is None else a if b is None else (b if sel else a)
                half, bit = half // 2, bit - 1
            row = cand[0]
        data = items.get(j * num_per + row) if row is not None else None
        if data is not None:
            chunk = np.asarray(data, dtype=np.uint8)[s * bpc:(s + 1) * bpc]
            out[s, :chunk.size] = chunk
    return out.reshape(-1)


def entry(db_idx, data):
    """One /update-row entry: [u32 BE chunk_len][u32 BE db_idx][data]."""
    data = bytes(data) if isinstance(data, (bytes, bytearray)) else np.asarray(data, dtype=np.uint8).tobytes()
    return (4 + len(data)).to_bytes(4, "big") + int(db_idx).to_bytes(4, "big") + data
