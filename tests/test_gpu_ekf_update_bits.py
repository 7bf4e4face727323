"""ovb_ekf_update's covariance and correction, bit for bit, at the tile edges of the EKF products (csrc/k_ekf.cu).

k_ekf_gemm1 (M = P[:, cols] H', S = H M[cols, :] + sigma^2 I) and k_ekf_downdate1 (P <- sym(P - Y Y'), dx = Y w) fix
the floating-point order of every output: one fused multiply-add chain over ascending k from zero. Whatever tiling or
arithmetic unit the kernels use, P and dx must keep the bits they had, so this module pins SHA-256 digests of them.

Cases: every (r, n) with r, n in EDGES (rows r > n are compressed by CholeskyQR2 first), at an even and an odd
max_state (they select different factor kernels, tests/ekf_routes.py), with sigma^2 and with per-row Rdiag. One digest
per (max_state, noise, n) covers P and dx of all r at that n, in order.

The digests were taken on an H100 80GB HBM3 from the build before the products were moved to the FP64 tensor cores.
`python -m tests.test_gpu_ekf_update_bits` prints them for the current build.
"""
import hashlib
import json

import numpy as np
import pytest

from open_vins_b200 import capi

EDGES = (1, 7, 8, 31, 32, 33, 64, 153, 154, 159, 160)
STATES = ((256, 194), (255, 177))  # (max_state, N): even and odd covariance pitch; N is off every 8 and 16 boundary
NOISES = ("sigma2", "Rdiag")


def _case(N, r, n, seed):
    rng = np.random.default_rng(seed)
    A = rng.standard_normal((N, N + 8))
    P = A @ A.T / (N + 8) + 0.1 * np.eye(N)
    cols = rng.permutation(N)[:n]  # one-column variables in a scattered order: the products gather P's rows through them
    H = rng.standard_normal((r, n))
    res = 0.1 * rng.standard_normal(r)
    Rdiag = rng.uniform(0.5, 2.0, r)
    return P, cols, H, res, Rdiag


def digests(eng, max_state, N, noise, n):
    h = hashlib.sha256()
    for r in EDGES:
        P, cols, H, res, Rdiag = _case(N, r, n, seed=1000 * r + n)
        eng.cov_set(P)
        kw = dict(sigma2=0.37) if noise == "sigma2" else dict(Rdiag=Rdiag)
        st, dx = eng.ekf_update(cols, np.ones(n, dtype=np.int32), H, res, **kw)
        assert st == 0, (max_state, noise, r, n, st)
        h.update(np.ascontiguousarray(eng.cov_get()).tobytes())
        h.update(np.ascontiguousarray(dx[:N]).tobytes())
    return h.hexdigest()


def _key(max_state, noise, n):
    return f"{max_state}/{noise}/n{n}"


# SHA-256 of P then dx after each update, for r in EDGES in order
DIGESTS = {
    "256/sigma2/n1": "da523d435e892897d5256f760bfdc42b1caa72ed078a160bd9f32005f5add292",
    "256/sigma2/n7": "aeec5293646e305f0f319fe5385a5c85c3b99664f9b55514643ce54dfd48903d",
    "256/sigma2/n8": "e8e00d1d6856a4b06a8db3b94b1a2057e0b24de62de4b32f9e542b1fdf215190",
    "256/sigma2/n31": "6ead7898e5d96959c63bdf53509b2a2fee5ebea56c34747a9c8fec6d901b1d67",
    "256/sigma2/n32": "131b98bb5d04c6168d05803c2c8127c983cac8f8fdb7b5795edafda5c994aa65",
    "256/sigma2/n33": "cec2f1300683efbeee85d30d073433ff6f83febf6930d3b09e2d9703e8ddb3c9",
    "256/sigma2/n64": "ea9c438d90bf4a2fbc1510d181a76caeedcbe55781d95e3c259e7bbf24c8bc9e",
    "256/sigma2/n153": "383698477d967ca8afdcf8dbce687c28ab337a41e036ebdd53aa258f42f07a70",
    "256/sigma2/n154": "0d324b2124b3325595706cd17c183f5de6cd7f9825fbf1bbd38924dda6a4d44a",
    "256/sigma2/n159": "f9edcac3c2edfdc69918ebe3f5e96ab77fb02b63ba1d7bccfb7bcd4c8079ef02",
    "256/sigma2/n160": "516983af6a1c36cc4752e7153572aca2051a35ccf63f7845fd1491acecd2f4d9",
    "256/Rdiag/n1": "af4272fadf8bf4bf7428e5229177377309ca1f7a65a2da41201e5dfdb49f3371",
    "256/Rdiag/n7": "0a5a62bf5bd62fcc572e20f83acd6e72d6ac91e8df352d6e29efef370a955ad0",
    "256/Rdiag/n8": "b4af8f2311801fab0866c0bdf7d489144ed3d0cdbfa7adb6bbe01c347c790378",
    "256/Rdiag/n31": "529c0fcabb3dfb7859ab0390809baeb47c374159f5d35e34df34adde6b9dc5a5",
    "256/Rdiag/n32": "918c54d9f391a49c4a60ebd9454ea1f56fdafead8b55532d03c2168daf35a5b2",
    "256/Rdiag/n33": "9bd847a8fbe35de745764d086541dd90149c30a1f76c9edeb34466544fbb6811",
    "256/Rdiag/n64": "a13813af373f8253388a94b6a90c45c58a6d349eb7783ac8d2abba97d7fc6663",
    "256/Rdiag/n153": "0e3e171daf405428c7e3fbdc0037f2655ef93fcabb5b4916828521a207388695",
    "256/Rdiag/n154": "7e5ab646518b46c789388a954a7e3d9fe9d9daab0dcff9be83c1704532ea08d6",
    "256/Rdiag/n159": "3b63283abac4aee03b89f3d13d80b40907cb34ebcb109eb1d95fe4dd4dddd178",
    "256/Rdiag/n160": "16f38b589c53d4b924193f0f366aea7d393791558d300e6505eb6191fac36751",
    "255/sigma2/n1": "2eeb11ddcad141bfae48ab9ef80a639bf4f9420dfd9225494e592b0a62777aa1",
    "255/sigma2/n7": "e42d1f6f59dbed97ec80a8c7b9bb1e71f4241a7e08190e56424499816c282aeb",
    "255/sigma2/n8": "74951333467549f7cd38991a750a3077b4e1029c109c42fb5e59ef58c5420aea",
    "255/sigma2/n31": "74b2276bfd07d02d6a546f91481abd982fe625ca44fe0cbd352fd56e37d007e8",
    "255/sigma2/n32": "ac0da42aca9f2b937c2ca34a2729bb78d00736be2e50ed26574615f70ba2f89f",
    "255/sigma2/n33": "25a5c4947810207a22b8ffcbd7157c40ddbcc2b3eaf783a750a589a3d48144d2",
    "255/sigma2/n64": "4c5355afd6a26bd7a663f88d237019f05b4517bbc161a6d62397ed412c1ad7b7",
    "255/sigma2/n153": "5a68b1d2ce32c4fdba7ae4d0a1e81f31436fcbd81e1a64e5ad8fed439c243e9b",
    "255/sigma2/n154": "5c8a5efbe4b206b54e76999835e33be48b778f85d382a8db2fa2af1a17b79091",
    "255/sigma2/n159": "0a8f3eecc228ec6416d5dffb4bea191df67bb0c32323da01790866502ec5f565",
    "255/sigma2/n160": "1a794e10d632c1d8728f55db2ec1dc4e2d5f350900d3611430c548739dd97577",
    "255/Rdiag/n1": "d3c9b8e268eb487bb48cab76f3516d1f5db9a4abf0649d46940f6261af0fb009",
    "255/Rdiag/n7": "684ee5d323d82f2dee75253e068a82eee2f5c685fe6f9774b8cc574e781e2767",
    "255/Rdiag/n8": "d77dfcaa7aea664f4b8ad327ad002ffe6f26810896e5df3c1536565bd0d6c5b6",
    "255/Rdiag/n31": "58938013572dcc2145bcf7e7d54d2a110a208ac53f7c7862f96153608bbe3c24",
    "255/Rdiag/n32": "456222f3bb9764d3e9b0c05b8aec19277ff333c5bfad55d2d005b3298013fdb9",
    "255/Rdiag/n33": "c0f8ab77c9702db697339da9eb54fbb5ef004296c40988f65eee8d3e1f62c201",
    "255/Rdiag/n64": "0f03a5f13a07931880b764a7f7d22a35a1dcc32c791746b2577b26eea37e244f",
    "255/Rdiag/n153": "ca5843b3efad611fa0102315ea732e69c1102543a8cfca734b19e9c543a59a0c",
    "255/Rdiag/n154": "ea7f0e1cb9335c084bd6ca7abe5824446e1e123f79e146aa2c3cf25a73b8e855",
    "255/Rdiag/n159": "dd19f32a28d60b075fecf10b591468550b64a533eacba0fdba47cc72dcfd3cf3",
    "255/Rdiag/n160": "d6903bd3108a3fea025a7eee82c64d4cbb7790fa97102b31c5f40ec3fefc268e",
}


@pytest.fixture(scope="module")
def engines():
    made = {ms: capi.Engine(max_state=ms, max_feats=16, max_meas=1024, max_rows=1024) for ms, _ in STATES}
    yield made
    for e in made.values():
        e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("n", EDGES)
@pytest.mark.parametrize("noise", NOISES)
@pytest.mark.parametrize("max_state,N", STATES)
def test_ekf_update_bits_unchanged(engines, max_state, N, noise, n):
    assert digests(engines[max_state], max_state, N, noise, n) == DIGESTS[_key(max_state, noise, n)]


if __name__ == "__main__":
    out = {}
    for ms, N in STATES:
        eng = capi.Engine(max_state=ms, max_feats=16, max_meas=1024, max_rows=1024)
        for noise in NOISES:
            for n in EDGES:
                out[_key(ms, noise, n)] = digests(eng, ms, N, noise, n)
        eng.close()
    print(json.dumps(out, indent=4))
