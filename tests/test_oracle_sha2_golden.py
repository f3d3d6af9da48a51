"""Pins the SHA-2 oracle of the GPU tests (python's hashlib) against the golden vectors of tests/golden/sha2_golden.py:
the FIPS 180-4 example messages and the inputs of the reference's HashTest.java."""
import hashlib

import pytest

from golden import sha2_golden as G

BITS = (224, 256, 384, 512)


@pytest.mark.parametrize("case", G.NIST, ids=[c["name"] for c in G.NIST])
def test_hashlib_reproduces_nist_examples(case):
    for bits in BITS:
        assert hashlib.new(f"sha{bits}", case["input"].encode("utf-8")).hexdigest() == case["digests"][bits]


@pytest.mark.parametrize("bits", BITS)
def test_hashlib_reproduces_java_inputs(bits):
    got = [None if s is None else hashlib.new(f"sha{bits}", s.encode("utf-8")).hexdigest() for s in G.JAVA_INPUTS]
    assert got == G.JAVA_DIGESTS[bits]


def test_golden_shapes():
    assert len(G.JAVA_INPUTS) == 11 and G.JAVA_INPUTS[0] is None
    # the padding cases of HashTest.java: 56, 63 and 64 bytes, and a multi-block string
    assert [len(G.JAVA_INPUTS[i]) for i in (3, 4, 5)] == [56, 63, 64] and len(G.JAVA_INPUTS[6]) > 128
    for bits in BITS:
        assert all(d is None or len(d) == bits // 4 for d in G.JAVA_DIGESTS[bits])
