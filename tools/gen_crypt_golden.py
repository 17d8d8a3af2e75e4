"""Writes tests/golden/chacha20poly1305.json: RFC 8439 test vectors (§2.4.2, §2.5.2, A.3, §2.6.2, §2.8.2),
each checked here against the `cryptography` package before it is written, and record-sized AEAD cases
sealed by `cryptography` from seeded messages.  Messages up to 65 bytes are stored whole; larger ones as
their seed and the SHA-256 of ciphertext || tag.

Usage: python tools/gen_crypt_golden.py   (needs `cryptography`; the tests only read the JSON)
"""
from __future__ import annotations

import hashlib
import json
import os
import random

from cryptography.hazmat.primitives import poly1305
from cryptography.hazmat.primitives.ciphers import Cipher, algorithms
from cryptography.hazmat.primitives.ciphers.aead import ChaCha20Poly1305

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "chacha20poly1305.json")
SUNSCREEN = (b"Ladies and Gentlemen of the class of '99: If I could offer you only one tip for the future, "
             b"sunscreen would be it.")
H = bytes.fromhex


def chacha20(key, counter, nonce, data):
    c = Cipher(algorithms.ChaCha20(key, counter.to_bytes(4, "little") + nonce), mode=None).encryptor()
    return c.update(data)


def message(seed: int, n: int, ff: bool) -> bytes:
    return b"\xff" * n if ff else random.Random(seed).randbytes(n)


def main() -> None:
    key = bytes(range(32))
    key80 = bytes(range(0x80, 0xA0))
    v = {"chacha20": [], "poly1305": [], "keygen": [], "aead": [], "records": []}
    # §2.4.2
    ct = H("6e2e359a2568f98041ba0728dd0d6981e97e7aec1d4360c20a27afccfd9fae0bf91b65c5524733ab8f593dabcd62b357"
           "1639d624e65152ab8f530c359f0861d807ca0dbf500d6a6156a38e088a22b65e52bc514d16ccf806818ce91ab7793736"
           "5af90bbf74a35be6b40b8eedf2785e42874d")
    v["chacha20"].append({"name": "RFC8439 2.4.2", "key": key.hex(), "nonce": "000000000000004a00000000",
                          "counter": 1, "plaintext": SUNSCREEN.hex(), "ciphertext": ct.hex()})
    # §2.5.2 and A.3
    polys = [("RFC8439 2.5.2", "85d6be7857556d337f4452fe42d506a80103808afb0db2fd4abff6af4149f51b",
              b"Cryptographic Forum Research Group".hex(), "a8061dc1305136c6c22b8baf0c0127a9"),
             ("RFC8439 A.3 #1", "00" * 32, "00" * 64, "00" * 16),
             ("RFC8439 A.3 #5", "02" + "00" * 31, "ff" * 16, "03" + "00" * 15),
             ("RFC8439 A.3 #6", "02" + "00" * 15 + "ff" * 16, "02" + "00" * 15, "03" + "00" * 15),
             ("RFC8439 A.3 #7", "01" + "00" * 31, "ff" * 16 + "f0" + "ff" * 15 + "11" + "00" * 15, "05" + "00" * 15),
             ("RFC8439 A.3 #8", "01" + "00" * 31, "ff" * 16 + "fb" + "fe" * 15 + "01" * 16, "00" * 16),
             ("RFC8439 A.3 #9", "02" + "00" * 31, "fd" + "ff" * 15, "fa" + "ff" * 15)]
    for name, k, m, tag in polys:
        p = poly1305.Poly1305(H(k))
        p.update(H(m))
        assert p.finalize() == H(tag), name
        v["poly1305"].append({"name": name, "key": k, "msg": m, "tag": tag})
    # §2.6.2
    kg = H("8ad5a08b905f81cc815040274ab29471a833b637e3fd0da508dbb8e2fdd1a646")
    assert chacha20(key80, 0, H("000000000001020304050607"), b"\0" * 32) == kg
    v["keygen"].append({"name": "RFC8439 2.6.2", "key": key80.hex(), "nonce": "000000000001020304050607",
                        "poly_key": kg.hex()})
    assert chacha20(key, 1, H("000000000000004a00000000"), SUNSCREEN) == ct
    # §2.8.2
    aead_ct = H("d31a8d34648e60db7b86afbc53ef7ec2a4aded51296e08fea9e2b5a736ee62d63dbea45e8ca9671282fafb69da92728b"
                "1a71de0a9e060b2905d6a5b67ecd3b3692ddbd7f2d778b8c9803aee328091b58fab324e4fad675945585808b4831d7bc"
                "3ff4def08e4b7a9de576d26586cec64b6116")
    aead_tag = H("1ae10b594f09e26a7e902ecbd0600691")
    nonce = H("070000004041424344454647")
    aad = H("50515253c0c1c2c3c4c5c6c7")
    assert ChaCha20Poly1305(key80).encrypt(nonce, SUNSCREEN, aad) == aead_ct + aead_tag
    v["aead"].append({"name": "RFC8439 2.8.2", "key": key80.hex(), "nonce": nonce.hex(), "aad": aad.hex(),
                      "plaintext": SUNSCREEN.hex(), "sealed": (aead_ct + aead_tag).hex()})
    # record-sized cases: the sizes a sealed file's records and headers take
    sizes = [0, 1, 15, 16, 17, 63, 64, 65, 24 + 4096, 24 + 65536 + 1024, 24 + (1 << 20) + 1024]
    for j, n in enumerate(sizes):
        for ff in (False, True):
            seed = 1000 + 2 * j + ff
            rng = random.Random(seed ^ 0x5EA1)
            k, nc, ad = rng.randbytes(32), rng.randbytes(12), rng.randbytes(24)
            m = message(seed, n, ff)
            sealed = ChaCha20Poly1305(k).encrypt(nc, m, ad)
            case = {"seed": seed, "ff": ff, "len": n, "key": k.hex(), "nonce": nc.hex(), "aad": ad.hex()}
            if n <= 65:
                case.update(plaintext=m.hex(), sealed=sealed.hex())
            else:
                case["sha256"] = hashlib.sha256(sealed).hexdigest()
            v["records"].append(case)
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    with open(OUT, "w") as f:
        json.dump(v, f, indent=1)
        f.write("\n")
    print("wrote", OUT)


if __name__ == "__main__":
    main()
