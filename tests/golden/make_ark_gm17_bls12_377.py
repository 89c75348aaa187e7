#!/usr/bin/env python3
"""Regenerate tests/golden/ark_gm17_bls12_377.json: four GM17 proofs on BLS12-377 made by ark, with their verifying keys.

Data only, copied from the ZoKrates repository (pass its checkout as the argument):
  * zokrates_stdlib/tests/tests/snark/gm17.json: proof.json and verification.key in hex, 3 public inputs.  Made by
      zokrates compile -i program.zok --curve bls12_377          (def main(field a, field b) -> field { return a + b; })
      zokrates setup --proving-scheme gm17 --backend ark
      zokrates compute-witness -a 1 2
      zokrates generate-proof --proving-scheme gm17 --backend ark
  * zokrates_core_test/tests/tests/snark/snark_verify_bls12_377_{1,2,5}.json: 1, 2 and 5 public inputs, made by
      zokrates compile -i ./circuit.zok -c bls12_377
      zokrates compute-witness
      zokrates setup -b ark -s gm17
      zokrates generate-proof -b ark -s gm17
    and flattened to decimals: every 0x... of proof.json (a, b, c, then the inputs), then of verification.key (h, g_alpha,
    h_beta, g_gamma, h_gamma, query).  Their first value list is the 8 proof coordinates, the second the inputs, the third
    the key.  This script turns them back into points in proof.json / verification.key form.

G2 coordinates are (c0, c1) pairs, as in ark's JSON.
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
FQ, FR = 48, 32


def hx(v, n):
    return "0x" + int(v).to_bytes(n, "big").hex()


def g1(f):
    return [hx(f[0], FQ), hx(f[1], FQ)]


def g2(f):
    return [[hx(f[0], FQ), hx(f[1], FQ)], [hx(f[2], FQ), hx(f[3], FQ)]]


def from_flat(proof, inputs, vk):
    proof, vk = [int(x) for x in proof], [int(x) for x in vk]
    assert len(proof) == 8 and len(vk) == 16 + 2 * (len(inputs) + 1)
    return {"proof": {"a": g1(proof[0:2]), "b": g2(proof[2:6]), "c": g1(proof[6:8])},
            "inputs": [hx(int(x), FR) for x in inputs],
            "vk": {"h": g2(vk[0:4]), "g_alpha": g1(vk[4:6]), "h_beta": g2(vk[6:10]), "g_gamma": g1(vk[10:12]),
                   "h_gamma": g2(vk[12:16]), "query": [g1(vk[i:i + 2]) for i in range(16, len(vk), 2)]}}


def main(ref):
    out = []
    src = "zokrates_stdlib/tests/tests/snark/gm17.json"
    proof, vk = json.load(open(os.path.join(ref, src)))["tests"][0]["input"]["values"]
    keys = ("h", "g_alpha", "h_beta", "g_gamma", "h_gamma", "query")
    out.append({"source": src, "proof": proof["proof"], "inputs": proof["inputs"], "vk": {k: vk[k] for k in keys}})
    for k in (1, 2, 5):
        src = "zokrates_core_test/tests/tests/snark/snark_verify_bls12_377_%d.json" % k
        proof, inputs, vk = json.load(open(os.path.join(ref, src)))["tests"][0]["input"]["values"]
        out.append(dict(source=src, **from_flat(proof, inputs, vk)))
    with open(os.path.join(HERE, "ark_gm17_bls12_377.json"), "w") as f:
        json.dump({"curve": "bls12_377", "scheme": "gm17", "proofs": out}, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main(sys.argv[1])
