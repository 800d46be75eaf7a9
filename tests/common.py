import hashlib
import json
import os

HERE = os.path.dirname(os.path.abspath(__file__))


def golden_vectors():
    with open(os.path.join(HERE, "golden", "reference_vectors.json")) as f:
        return json.load(f)["vectors"]


def sha(b) -> str:
    return hashlib.sha256(bytes(b)).hexdigest()


def with_text_chunk(png: bytes, payload_len: int) -> bytes:
    """inserts a valid ancillary chunk in front of fdEC: moves the zlib stream to another byte alignment (Stream::bit0)"""
    import zlib
    body = bytes(range(65, 65 + payload_len))
    ch = len(body).to_bytes(4, "big") + b"tEXt" + body + (zlib.crc32(b"tEXt" + body) & 0xFFFFFFFF).to_bytes(4, "big")
    return png[:33] + ch + png[33:]
