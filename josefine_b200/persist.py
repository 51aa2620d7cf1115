"""Chain records in josefine's on-disk vocabulary (SURVEY.md section 8f, row 4) -- logical level only.

The reference keeps each node's chain in a sled tree (src/raft/chain.rs:99-104):
  * one record per block: key = the BlockId's 8 big-endian bytes (chain.rs:63-66), value =
    `bincode::serialize(&Block{id, next, data})` (chain.rs:139-153, 160-176, 178-193);
  * the key b"commit" -> the committed BlockId's 8 bytes, written by `Chain::commit`
    (chain.rs:195-205) and read back by `Chain::new` (chain.rs:117-136), which reopens with
    head = commit and the id generator at commit.

bincode 1.3 (default options: fixed-width little-endian integers, u64 lengths) of the derives:
  BlockId(Bytes) via `serialize_bytes`  ->  u64 len (=8) + 8 bytes
  Vec<u8>                                ->  u64 len + bytes
so a Block record is  08 00.. | id_be8 | 08 00.. | next_be8 | len_le8 | data.

What this module does: turn replicas' device-resident block tables (`jr_chain_export_many`) into that
ordered (key, value) record list and back (`jr_node_restart_many`).  What it does NOT do: write sled's own page/log file
format (sled 0.34.7 is a third-party dependency that is not vendored in the reference, and
its file layout is not something to restate from memory) -- a josefine-side loader is one
`db.insert(k, v)` loop over these records.  **Parity unpinned**: no Rust toolchain here, the byte
layout is derived from the bincode specification; tests/test_persist.py pins the derivation.

Record order is sled's: lexicographic by key, which puts b"commit" (0x63...) after every block key
whose first byte is below 0x63 -- the keyspace collision behind deviation D6 (DESIGN.md).
"""
from __future__ import annotations

import struct
from typing import Dict, Iterable, List, Optional, Tuple

COMMIT_KEY = b"commit"


def block_key(block_id: int) -> bytes:
    return block_id.to_bytes(8, "big")


def encode_block(block_id: int, next_id: int, data: bytes) -> bytes:
    """bincode::serialize(&Block) -- chain.rs:86-91."""
    return (struct.pack("<Q", 8) + block_key(block_id) + struct.pack("<Q", 8) + block_key(next_id) +
            struct.pack("<Q", len(data)) + bytes(data))


def decode_block(value: bytes) -> Tuple[int, int, bytes]:
    def take(off: int) -> Tuple[bytes, int]:
        if off + 8 > len(value):
            raise ValueError("truncated bincode record")
        (n,) = struct.unpack_from("<Q", value, off)
        if off + 8 + n > len(value):
            raise ValueError("truncated bincode record")
        return value[off + 8:off + 8 + n], off + 8 + n
    idb, off = take(0)
    nxb, off = take(off)
    data, off = take(off)
    if len(idb) != 8 or len(nxb) != 8 or off != len(value):
        raise ValueError("not a Block record")
    return int.from_bytes(idb, "big"), int.from_bytes(nxb, "big"), data


def _records(commit: int, commit_key: bool, blocks, payloads: Optional[Dict[int, bytes]]) -> List[Tuple[bytes, bytes]]:
    recs = []
    for bid, nxt, tok in blocks:
        data = payloads[tok] if payloads is not None and tok in payloads else (struct.pack("<Q", tok) if tok else b"")
        recs.append((block_key(bid), encode_block(bid, nxt, data)))
    if commit_key:                          # the key only exists once Chain::commit has run (chain.rs:198)
        recs.append((COMMIT_KEY, block_key(commit)))
    recs.sort(key=lambda kv: kv[0])
    return recs


def export_many(api, targets: Iterable[Tuple[int, int]],
                payloads: Optional[Dict[int, bytes]] = None) -> Dict[Tuple[int, int], List[Tuple[bytes, bytes]]]:
    """`chain_records` of many replicas through one `chain_export_many` call: {(group, node): records}."""
    targets = list(targets)
    return {(g, n): _records(commit, ck, blocks, payloads)
            for (g, n), (commit, ck, blocks) in zip(targets, api.chain_export_many(targets))}


def chain_records(api, group: int, node: int, payloads: Optional[Dict[int, bytes]] = None) -> List[Tuple[bytes, bytes]]:
    """Every record josefine's sled tree would hold for replica (group, node), in sled's key order.

    `payloads` maps the engine's 64-bit block tokens to the payload bytes the host kept (deviation D5);
    a token without an entry is written as its own 8 little-endian bytes so the record stays reversible.
    """
    return export_many(api, [(group, node)], payloads)[(group, node)]


def reopen(records: Iterable[Tuple[bytes, bytes]]) -> dict:
    """What `Chain::new` (chain.rs:117-136) sees in a tree holding `records`: commit (0 if the key is absent),
    head = commit, id_gen at commit, and the block records by id."""
    commit, blocks = 0, {}
    for k, v in records:
        if k == COMMIT_KEY:
            if len(v) != 8:
                raise ValueError("commit value is not 8 bytes (chain.rs:122 try_into().unwrap())")
            commit = int.from_bytes(v, "big")
        else:
            bid, nxt, data = decode_block(v)
            if block_key(bid) != k:
                raise ValueError("record key does not match the block id inside it")
            blocks[bid] = (nxt, data)
    return {"commit": commit, "head": commit, "id_gen": commit, "blocks": blocks}


def import_records(records: Iterable[Tuple[bytes, bytes]], tokens: Optional[Dict[bytes, int]] = None):
    """The arguments of `jr_node_restart` / `RaftApi.node_restart` for a node that reopens a tree holding `records`
    (chain.rs:117-137): (blocks, commit, commit_key) with blocks = [(id, next, token)].

    Payload bytes stay on the host (deviation D5): `tokens` maps payload bytes to the 64-bit token the host wants the
    engine to carry for them; a payload without an entry gets the token `chain_records` wrote for token-only payloads
    (its own 8 little-endian bytes) or, failing that, 0.
    """
    st = reopen(records)
    commit_key = any(k == COMMIT_KEY for k, _ in records) if not isinstance(records, dict) else False
    blocks = []
    for bid in sorted(st["blocks"]):
        nxt, data = st["blocks"][bid]
        if tokens is not None and data in tokens:
            tok = tokens[data]
        elif len(data) == 8:
            (tok,) = struct.unpack("<Q", data)
        else:
            tok = 0
        blocks.append((bid, nxt, tok))
    return blocks, st["commit"], commit_key


def restart_from_records(api, group: int, node: int, now_ms: int, records, tokens: Optional[Dict[bytes, int]] = None):
    """`RaftHandle::new` over an existing data directory: load a sled export back into replica (group, node)."""
    records = list(records)
    blocks, commit, commit_key = import_records(records, tokens)
    api.node_restart(group, node, now_ms, blocks, commit, commit_key)


def restart_many_from_records(api, now_ms: int, trees: Dict[Tuple[int, int], Iterable[Tuple[bytes, bytes]]],
                              tokens: Optional[Dict[bytes, int]] = None):
    """`RaftHandle::new` over many data directories at once: trees = {(group, node): records}, one
    `node_restart_many` call."""
    chains = []
    for (g, n), records in trees.items():
        blocks, commit, commit_key = import_records(list(records), tokens)
        chains.append((g, n, blocks, commit, commit_key))
    api.node_restart_many(now_ms, chains)
