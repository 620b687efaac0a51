"""Generates tests/golden/ordered_roots.json from the reference's own ordered-root tests
(crates/ethereum/primitives/src/receipt.rs:180-245: check_transaction_root, check_withdrawals_root,
check_receipt_root_optimism).  Run against a checkout of reth (the tests only read the generated file):

    python tests/golden/make_ordered_roots.py /path/to/reth

The block fixtures there are RLP blocks whose headers carry the expected roots; the items are the raw encodings found
in the block body (what the encoder closure of ordered_trie_root_with_encoder writes for legacy transactions and
withdrawals).  The receipt case is assembled from the field values the test states.
"""
import json
import os
import re
import sys

REL = "crates/ethereum/primitives/src/receipt.rs"
SRC = os.path.join(sys.argv[1] if len(sys.argv) > 1 else ".", REL)
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "ordered_roots.json")


def rlp_item(buf, pos):
    """-> (is_list, payload_start, payload_end, item_end) of the item at pos."""
    b = buf[pos]
    if b < 0x80:
        return False, pos, pos + 1, pos + 1
    if b < 0xB8:
        return False, pos + 1, pos + 1 + (b - 0x80), pos + 1 + (b - 0x80)
    if b < 0xC0:
        ll = b - 0xB7
        n = int.from_bytes(buf[pos + 1:pos + 1 + ll], "big")
        return False, pos + 1 + ll, pos + 1 + ll + n, pos + 1 + ll + n
    if b < 0xF8:
        return True, pos + 1, pos + 1 + (b - 0xC0), pos + 1 + (b - 0xC0)
    ll = b - 0xF7
    n = int.from_bytes(buf[pos + 1:pos + 1 + ll], "big")
    return True, pos + 1 + ll, pos + 1 + ll + n, pos + 1 + ll + n


def list_items(buf, pos):
    """raw encodings of the children of the list at pos"""
    is_list, a, b, _ = rlp_item(buf, pos)
    assert is_list
    out = []
    while a < b:
        _, _, _, e = rlp_item(buf, a)
        out.append((a, e))
        a = e
    assert a == b
    return out


def payload(buf, span):
    _, a, b, _ = rlp_item(buf, span[0])
    return buf[a:b]


def rlp_bytes(x: bytes) -> bytes:
    if len(x) == 1 and x[0] < 0x80:
        return x
    if len(x) < 56:
        return bytes([0x80 + len(x)]) + x
    ll = (len(x).bit_length() + 7) // 8
    return bytes([0xB7 + ll]) + len(x).to_bytes(ll, "big") + x


def rlp_list(items) -> bytes:
    body = b"".join(items)
    if len(body) < 56:
        return bytes([0xC0 + len(body)]) + body
    ll = (len(body).bit_length() + 7) // 8
    return bytes([0xF7 + ll]) + len(body).to_bytes(ll, "big") + body


def rlp_uint(v: int) -> bytes:
    return rlp_bytes(v.to_bytes((v.bit_length() + 7) // 8, "big"))


def main():
    text = open(SRC).read()
    cases = []

    def block_hexes(fn_name):
        body = text[text.index(f"fn {fn_name}()"):]
        body = body[:body.index("\n    }\n")]
        return [bytes.fromhex(h) for h in re.findall(r'hex!\(\s*"([0-9a-f]+)"', body)], body

    blocks, _ = block_hexes("check_transaction_root")
    blk = blocks[0]
    top = list_items(blk, 0)
    header = list_items(blk, top[0][0])
    txs = list_items(blk, top[1][0])
    cases.append({"name": "check_transaction_root", "ref": "receipt.rs:180-190", "field": "transactions_root",
                  "items": [blk[a:b].hex() for a, b in txs], "root": payload(blk, header[4]).hex()})

    blocks, _ = block_hexes("check_withdrawals_root")
    for k, blk in enumerate(blocks):
        top = list_items(blk, 0)
        header = list_items(blk, top[0][0])
        ws = list_items(blk, top[3][0])
        cases.append({"name": f"check_withdrawals_root[{k}]", "ref": "receipt.rs:192-217", "field": "withdrawals_root",
                      "items": [blk[a:b].hex() for a, b in ws], "root": payload(blk, header[16]).hex()})

    _, body = block_hexes("check_receipt_root_optimism")
    bloom = bytes.fromhex(re.search(r'bloom!\(\s*"([0-9a-f]+)"', body).group(1))
    gas = int(re.search(r"cumulative_gas_used: (\d+)", body).group(1))
    root = re.search(r'b256!\("0x([0-9a-f]{64})"\)', body).group(1)
    assert "TxType::Eip2930" in body and "success: true" in body and "Address::ZERO" in body
    log = rlp_list([rlp_bytes(bytes(20)), rlp_list([]), rlp_bytes(b"")])
    receipt = b"\x01" + rlp_list([rlp_uint(1), rlp_uint(gas), rlp_bytes(bloom), rlp_list([log])])
    cases.append({"name": "check_receipt_root_optimism", "ref": "receipt.rs:218-244", "field": "receipts_root",
                  "items": [receipt.hex()], "root": root})

    json.dump({"source": REL, "cases": cases}, open(OUT, "w"), indent=1)
    print(f"wrote {OUT}: {len(cases)} cases")


if __name__ == "__main__":
    main()
