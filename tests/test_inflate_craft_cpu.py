"""CPU: the DEFLATE crafting helper (tests/deflate_craft.py) and its cases (tests/inflate_cases.py) checked against
zlib, so that the device decoder tests (tests/test_gpu_x_inflate_edges.py) compare with what the cases claim."""
import zlib

import pytest

from tests import deflate_craft as D
from tests import inflate_cases as IC


def test_bit_writer_is_lsb_first_and_codes_msb_first():
    w = D.BitWriter()
    w.put(1, 1)
    w.put(0b10, 2)
    w.put_code(0b0011, 4)          # sent 0, 0, 1, 1: bits 3..6
    assert w.bit_len == 7 and w.getvalue() == bytes([0b1100101])
    w.align()
    w.put_bytes(b"\xab")
    assert w.getvalue() == bytes([0b1100101, 0xAB])


def test_canonical_codes_are_rfc1951s_example():
    lens = [3, 3, 3, 3, 3, 2, 4, 4]  # RFC 1951 3.2.2: A..H
    codes = D.canonical(lens)
    assert [codes[s][0] for s in range(8)] == [0b010, 0b011, 0b100, 0b101, 0b110, 0b00, 0b1110, 0b1111]


@pytest.mark.parametrize("k", [2, 3, 5, 16, 19, 200, 286])
def test_complete_and_skewed_lengths_are_complete(k):
    assert D.kraft(D.complete_lengths(range(k), 300)) == 1.0
    if k <= 16:  # noqa: PLR2004
        assert D.kraft(D.skewed_lengths(list(range(k)), k)) == 1.0


def test_hand_written_blocks_equal_zlib_output():
    data = b"hello, hello, hello world\n" * 20
    tokens = list(data[:26]) + [D.Match(258, 26), D.Match(len(data) - 26 - 258, 26)]
    for build in (lambda w: D.fixed(w, tokens), lambda w: D.dynamic_for(tokens, w=w),
                  lambda w: D.stored(w, data)):
        w = D.BitWriter()
        build(w)
        assert zlib.decompress(w.getvalue(), -15) == data


@pytest.mark.parametrize("name", sorted(IC.VALID))
def test_every_valid_case_inflates_with_zlib_to_its_bytes(name):
    blocks = IC.VALID[name]()
    n = 0
    for b in blocks:
        for payload, crc, isize in D.split_bgzf(b):
            out = D.host_rule(payload, isize, crc)
            assert out is not None, name
            d = zlib.decompressobj(-15)
            assert d.decompress(payload) == out and d.eof and not d.unused_data
            n += 1
    assert n == len(blocks)


def test_the_valid_cases_have_the_shapes_they_name():
    def header(payload):  # HLIT, HDIST, HCLEN of a stream that starts with a dynamic block
        v = int.from_bytes(payload[:3], "little")
        assert v & 7 in (4, 5)  # noqa: PLR2004
        return ((v >> 3) & 31) + 257, ((v >> 8) & 31) + 1, ((v >> 13) & 15) + 4

    first = lambda name, i=0: D.split_bgzf(IC.VALID[name]()[i])[0]  # noqa: E731
    assert header(first("long_codes")[0]) == (266, 16, 19)
    assert header(first("literal_only")[0])[:2] == (257, 1)
    assert header(first("hclen_five")[0]) == (257, 1, 5)
    assert header(first("repeats")[0])[:2] == (260, 8)
    assert [header(first("single_distance_code", i)[0])[1] for i in (0, 1)] == [1, 4]
    payload, _, isize = first("isize_65536")
    assert isize == 65536  # noqa: PLR2004
    sizes = [len(b) for b in IC.VALID["stored_at_bit_offsets"]()]
    assert max(sizes) == 65536  # noqa: PLR2004
    assert [isize for _, _, isize in map(lambda b: D.split_bgzf(b)[0], IC.VALID["empty_block_in_the_middle"]())][1] == 0


@pytest.mark.parametrize("name", sorted(IC.refusal_cases()))
def test_every_refusal_is_refused_by_the_host_rule_with_zlibs_message(name):
    block, code, msg = IC.refusal_cases()[name]
    (payload, crc, isize), = D.split_bgzf(block)
    assert D.host_rule(payload, isize, crc) is None
    err = D.zlib_error(payload)
    if msg is None:  # the stream is valid: ISIZE or the CRC is what is wrong
        assert err is None and code in (IC.INF_OUTPUT_OVERRUN, IC.INF_SIZE_MISMATCH, IC.INF_BAD_CRC)
    else:
        assert err is not None and msg in err, err


def test_the_incomplete_code_length_code_of_the_report():
    block, code, _ = IC.refusal_cases()["cl_incomplete"]
    (payload, _, _), = D.split_bgzf(block)
    # the same stream with the code-length code made complete (0: 3 -> 0: 2) is the three A's
    w = D.BitWriter()
    lit = [0] * 257
    lit[65] = lit[256] = 1
    cl = [0] * 19
    cl[18], cl[1], cl[0] = 1, 2, 2
    D.dynamic(w, lit, [0], [65, 65, 65], cl_lens=cl,
              cl_symbols=[(18, 54), (1, 0), (18, 127), (18, 41), (1, 0), (0, 0)])
    assert zlib.decompress(w.getvalue(), -15) == b"AAA"
    assert D.kraft([1, 2, 3]) == 0.875 and code == IC.INF_BAD_CODE_LENGTHS  # noqa: PLR2004
