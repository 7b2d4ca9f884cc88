"""Crafted BGZF blocks for the device BGZF decoder (tests/deflate_craft.py): the valid shapes, each with the bytes it
inflates to, and the single-fault refusals, each with the decoder's INF_* code and zlib's message.  A valid case may
span several BGZF blocks (the test compares the concatenated output); a refusal is exactly one block."""
import random
import zlib

from tests import deflate_craft as D
from tests.deflate_craft import BitWriter, DSym, Match, Sym

# csrc/inflate.cuh
INF_OK, INF_BAD_BLOCK_TYPE, INF_BAD_STORED_LEN, INF_BAD_CODE_LENGTHS = 0, 1, 2, 3
INF_BAD_SYMBOL, INF_BAD_DISTANCE, INF_OUTPUT_OVERRUN, INF_INPUT_OVERRUN, INF_SIZE_MISMATCH, INF_BAD_CRC = 4, 5, 6, 7, 8, 9
BGZF_EOF = D.bgzf_block(b"\x03\x00")


def _rand(n: int, seed: int) -> bytes:
    return random.Random(seed).randbytes(n)


def _block(w: BitWriter, data: bytes) -> bytes:
    return D.bgzf_block(w.getvalue(), data)


def _fixed(tokens, history: bytes = b"") -> tuple[bytes, bytes]:
    w = BitWriter()
    D.fixed(w, tokens)
    data = D.expand(tokens, history)
    return w.getvalue(), data


def long_codes():
    lits = list(range(97, 110))
    lit_lens = D.skewed_lengths(lits + [257, 265, 256], 266)                   # 257: 14 bits, 265 and EOB: 15 bits
    dist_lens = D.skewed_lengths(list(range(15, -1, -1)), 16)                   # distance symbols 0 and 1: 15 bits
    tokens = lits + [Match(3, 1), Match(11, 2), Match(12, 5), 97, Match(12, 6), 109]
    w = BitWriter()
    D.dynamic(w, lit_lens, dist_lens, tokens, hclen=19)
    assert max(lit_lens) == max(dist_lens) == 15                                # noqa: PLR2004
    return [_block(w, D.expand(tokens))]


def single_distance_code():
    out = []
    for sym, dist in ((0, 1), (3, 4)):                                          # one code of length 1: HDIST 1 and 4
        dist_lens = [0] * sym + [1]
        tokens = [120, 121, 122, 123, Match(20, dist), 65]
        lit_lens = D.complete_lengths({120, 121, 122, 123, 65, 256, 269}, 270)  # 269: lengths 19..22
        w = BitWriter()
        D.dynamic(w, lit_lens, dist_lens, tokens)
        out.append(_block(w, D.expand(tokens)))
    return out


def literal_only():
    tokens = list(b"no distance codes at all\n")
    w = BitWriter()
    D.dynamic(w, D.complete_lengths(set(tokens) | {256}, 257), [0], tokens)     # HLIT 257, HDIST 1, all zero
    return [_block(w, bytes(tokens))]


def eob_only_block():
    w = BitWriter()
    D.stored(w, b"abc", final=False)
    lit_lens = [0] * 256 + [1]                                                  # the end-of-block code alone, 1 bit
    D.dynamic(w, lit_lens, [0], [])
    return [_block(w, b"abc")]


def hclen_five():
    lit_lens = [8] * 255 + [0, 8]                                               # literals 0..254 and EOB: 8 bits each
    tokens = list(range(255))
    w = BitWriter()
    D.dynamic(w, lit_lens, [0], tokens)                                         # HCLEN 5: the lengths of 16, 17, 18, 0, 8
    return [_block(w, bytes(tokens))]


def hlit_286_hdist_30():
    hist = _rand(25000, 1)
    w = BitWriter()
    D.stored(w, hist, final=False)
    tokens = [Match(258, 24600), Match(258, 30), 7, Match(3, 25000)]
    lit_lens = D.complete_lengths({7, 256, 257, 285}, 286)
    dist_lens = D.complete_lengths({29, 9, 28}, 30)
    D.dynamic(w, lit_lens, dist_lens, tokens)
    return [_block(w, hist + D.expand(tokens, hist))]


def repeats():
    lit_lens = [0] * 260
    lit_lens[65] = lit_lens[66] = 2
    lit_lens[256] = lit_lens[257] = lit_lens[258] = lit_lens[259] = 3
    dist_lens = [3] * 8
    cl = [(18, 65 - 11), (2, 0), (2, 0),
          (17, 0), (17, 7), (18, 127), (18, 0), (18, 27 - 11),                  # 17 x3, x10, 18 x138, x11, then x27
          (3, 0), (16, 3), (16, 2)]                                             # 16 x6 runs from 257..259 into distances 0..2
    assert 3 + 10 + 138 + 11 + 27 == 256 - 67                                   # noqa: PLR2004
    tokens = [65, 66, Match(3, 1), Match(4, 2), 66, 65, 65, 66, Match(5, 13), Match(5, 16), 65]
    w = BitWriter()
    D.dynamic(w, lit_lens, dist_lens, tokens, cl_symbols=cl)
    return [_block(w, D.expand(tokens))]


def length_symbols():
    hist = list(_rand(300, 2))
    tokens = list(hist)
    for i in range(28):
        lo, hi = D.LEN_BASE[i], D.LEN_BASE[i] + (1 << D.LEN_EXTRA[i]) - 1
        tokens += [Match(lo, 7 + i, lsym=257 + i), 5, Match(hi if i < 27 else 257, 290, lsym=257 + i), 6]  # noqa: PLR2004
    tokens += [Match(258, 1), 9, Match(258, 299, lsym=284), 10, Match(258, 2, lsym=284)]  # 258 as 285 and as 284 + 31
    payload, data = _fixed(tokens)
    return [D.bgzf_block(payload, data)]


def distances():
    out = []
    hist = list(_rand(40, 3))
    tokens = list(hist) + [Match(3, 1), Match(258, 1)]
    for d in range(2, 34):
        for n in sorted({d - 1, d, d + 1, 2 * d + 3, 31, 32, 33, 64, 100, 258} - {1, 2}):  # len < d, = d, > d
            tokens += [Match(n, d), d]
    payload, data = _fixed(tokens)
    out.append(D.bgzf_block(payload, data))
    return out


def word_copy_alignments():
    tokens = list(_rand(64, 4))
    op = 64
    for dst in range(8):
        for d in range(16, 24):
            while op % 8 != dst:
                tokens.append(op & 0xFF)
                op += 1
            n = 16 + (dst * 8 + d) % 41
            tokens.append(Match(n, d))
            op += n
    payload, data = _fixed(tokens)
    return [D.bgzf_block(payload, data)]


def far_and_first_byte():
    hist = _rand(33000, 5)
    w = BitWriter()
    D.stored(w, hist, final=False)
    tokens = [Match(258, 32768), 1, Match(100, 32768)]
    D.fixed(w, tokens)
    far = _block(w, hist + D.expand(tokens, hist))
    tokens = [1, 2, 3, 4, 5, Match(10, 5)] + list(range(6, 200)) + [Match(258, 209)]  # both read byte 0
    payload, data = _fixed(tokens)
    return [far, D.bgzf_block(payload, data)]


def stored_at_bit_offsets():
    out = []
    for bit in range(8):
        for size in (0, 1, None):
            w = BitWriter()
            lead = [144 + k for k in range((bit - 2) % 8)]                      # 9-bit literals: 3 + 9 m + 7 bits
            D.fixed(w, lead, final=False)
            assert w.bit_len % 8 == bit, (bit, w.bit_len)
            # the largest stored block in a BGZF block: payload = the bytes up to LEN, LEN, NLEN, data <= 65536 - 26
            n = 65510 - (w.bit_len + 3 + 7) // 8 - 4 if size is None else size
            data = _rand(n, 100 + bit)
            D.stored(w, data)
            out.append(D.bgzf_block(w.getvalue(), bytes(lead) + data))
    return out


def many_blocks():
    rng = random.Random(6)
    w, hist = BitWriter(), b""
    for k in range(36):
        kind = k % 3
        if kind == 0:
            data = bytes(rng.randrange(256) for _ in range(rng.randrange(0, 40)))
            D.stored(w, data, final=False)
            hist += data
            continue
        tokens = [rng.randrange(256) for _ in range(5)]
        if hist:
            for _ in range(6):
                tokens.append(Match(rng.randrange(3, 259), rng.randrange(1, len(hist) + 1)))
                tokens.append(rng.randrange(256))
        data = D.expand(tokens, hist)
        if kind == 1:
            D.fixed(w, tokens, final=False)
        else:
            D.dynamic_for(tokens, final=False, w=w)
        hist += data
    D.fixed(w, [10])
    hist += b"\n"
    return [_block(w, hist)]


def isize_65536():
    tokens = [97] + [Match(258, 1)] * 254 + [Match(3, 1)]
    payload, data = _fixed(tokens)
    assert len(data) == 65536                                                   # noqa: PLR2004
    return [D.bgzf_block(payload, data)]


def empty_block_in_the_middle():
    a, b = b"first\n" * 100, b"second\n" * 100
    return [D.bgzf_block(_raw(a), a), BGZF_EOF, D.bgzf_block(_raw(b), b)]


def _raw(data: bytes, level: int = 6, strategy: int = zlib.Z_DEFAULT_STRATEGY) -> bytes:
    c = zlib.compressobj(level, zlib.DEFLATED, -15, 8, strategy)
    return c.compress(data) + c.flush()


VALID = {f.__name__: f for f in (long_codes, single_distance_code, literal_only, eob_only_block, hclen_five,
                                 hlit_286_hdist_30, repeats, length_symbols, distances, word_copy_alignments,
                                 far_and_first_byte, stored_at_bit_offsets, many_blocks, isize_65536,
                                 empty_block_in_the_middle)}


def valid_cases() -> dict[str, list[bytes]]:
    """name -> BGZF blocks; each block's footer carries the ISIZE and CRC32 of its intended output."""
    return {name: f() for name, f in VALID.items()}


# ---------------------------------------------------------------------------------------------------------------
# single-fault refusals: name -> (BGZF block, INF_* code, zlib's message or None when the stream itself is valid)
# ---------------------------------------------------------------------------------------------------------------
def _dyn(tokens=(65, 66), **kw) -> bytes:
    w = BitWriter()
    lit = kw.pop("lit_lens", D.complete_lengths({65, 66, 256}, 257))
    dist = kw.pop("dist_lens", [0])
    D.dynamic(w, lit, dist, list(tokens), **kw)
    return w.getvalue()


def _fixed_payload(tokens, **kw) -> bytes:
    w = BitWriter()
    D.fixed(w, tokens, **kw)
    return w.getvalue()


def refusal_cases() -> dict[str, tuple[bytes, int, str | None]]:
    AB = b"AB"  # noqa: N806
    cases = {}

    def add(name, payload, data, code, msg, **kw):
        cases[name] = (D.bgzf_block(payload, data, **kw), code, msg)

    w = BitWriter()
    w.put(1, 1), w.put(3, 2), w.put(0, 16)
    add("block_type_3", w.getvalue(), b"x", INF_BAD_BLOCK_TYPE, "invalid block type")
    w = BitWriter()
    D.stored(w, b"abc", nlen=0xFFFC ^ 1)
    add("stored_nlen", w.getvalue(), b"abc", INF_BAD_STORED_LEN, "invalid stored block lengths")
    too_many = "too many length or distance symbols"
    for hlit in (287, 288):
        add(f"hlit_{hlit}", _dyn(hlit=hlit), AB, INF_BAD_CODE_LENGTHS, too_many)
    for hdist in (31, 32):
        add(f"hdist_{hdist}", _dyn(hdist=hdist), AB, INF_BAD_CODE_LENGTHS, too_many)
    cl_set, lit_set, dist_set = "invalid code lengths set", "invalid literal/lengths set", "invalid distances set"
    # the code-length code: over-subscribed, and incomplete ({18: 1, 1: 2, 0: 3}: Kraft sum 7/8)
    over_cl = [0] * 19
    for s in (0, 1, 2, 18):
        over_cl[s] = 1
    add("cl_oversubscribed", _dyn(cl_lens=over_cl, cl_symbols=[]), AB, INF_BAD_CODE_LENGTHS, cl_set)
    inc_cl = [0] * 19
    inc_cl[18], inc_cl[1], inc_cl[0] = 1, 2, 3
    lit = [0] * 257
    lit[65] = lit[256] = 1
    w = BitWriter()
    D.dynamic(w, lit, [0], [65, 65, 65], cl_lens=inc_cl,
              cl_symbols=[(18, 65 - 11), (1, 0), (18, 138 - 11), (18, 52 - 11), (1, 0), (0, 0)])
    add("cl_incomplete", w.getvalue(), b"AAA", INF_BAD_CODE_LENGTHS, cl_set)
    lit_over = D.complete_lengths({65, 66, 256}, 257)
    lit_over[67] = 1
    add("lit_oversubscribed", _dyn(tokens=(), lit_lens=lit_over, eob=False), AB, INF_BAD_CODE_LENGTHS, lit_set)
    lit_inc = D.complete_lengths({65, 66, 256, 67}, 257)
    lit_inc[67] = 0
    add("lit_incomplete", _dyn(lit_lens=lit_inc), AB, INF_BAD_CODE_LENGTHS, lit_set)
    lit_single2 = [0] * 256 + [2]                                               # one code, but of length 2
    add("lit_single_code_of_length_2", _dyn(tokens=(), lit_lens=lit_single2), b"", INF_BAD_CODE_LENGTHS, lit_set,
        isize=1)
    add("dist_oversubscribed", _dyn(dist_lens=[1, 1, 1]), AB, INF_BAD_CODE_LENGTHS, dist_set)
    add("dist_incomplete", _dyn(dist_lens=[2, 2]), AB, INF_BAD_CODE_LENGTHS, dist_set)
    add("dist_single_code_of_length_2", _dyn(dist_lens=[0, 2]), AB, INF_BAD_CODE_LENGTHS, dist_set)
    repeat = "invalid bit length repeat"
    lit = D.complete_lengths({65, 66, 256}, 257)
    cl = D.rle_lengths(lit + [0])
    assert cl[0] == (18, 65 - 11)                                               # symbols 0..64 are zero
    add("repeat_16_first", _dyn(cl_symbols=[(16, 0), (18, 62 - 11)] + cl[1:]), AB, INF_BAD_CODE_LENGTHS, repeat)
    add("repeat_17_past_the_end", _dyn(cl_symbols=cl[:-1] + [(17, 1)]), AB, INF_BAD_CODE_LENGTHS, repeat)
    add("repeat_18_past_the_end", _dyn(cl_symbols=cl[:-1] + [(18, 0)]), AB, INF_BAD_CODE_LENGTHS, repeat)
    add("repeat_16_past_the_end", _dyn(cl_symbols=cl[:-2] + [(2, 0), (16, 0)]), AB, INF_BAD_CODE_LENGTHS, repeat)
    no_eob = D.complete_lengths({65, 66}, 257)
    add("no_end_of_block_code", _dyn(lit_lens=no_eob, eob=False), AB, INF_BAD_CODE_LENGTHS,
        "invalid code -- missing end-of-block")
    hclen4 = [0] * 19
    hclen4[0] = hclen4[18] = 1
    add("hclen_4", _dyn(tokens=(), lit_lens=[0] * 257, eob=False, cl_lens=hclen4, cl_symbols=[(18, 127), (18, 119 - 11), (0, 0)]),
        AB, INF_BAD_CODE_LENGTHS, "invalid code -- missing end-of-block")
    for s in (286, 287):
        add(f"fixed_symbol_{s}", _fixed_payload([65, Sym(s)], eob=False), AB, INF_BAD_SYMBOL, "invalid literal/length code")
    for s in (30, 31):
        add(f"fixed_distance_{s}", _fixed_payload([65, Sym(257), DSym(s)], eob=False), b"AAAA", INF_BAD_DISTANCE,
            "invalid distance code")
    add("distance_one_too_far", _fixed_payload([65, 66, 67, Match(3, 4)]), b"ABCABC", INF_BAD_DISTANCE,
        "invalid distance too far back")
    tokens = list(b"twelve bytes")
    p = _fixed_payload(tokens)
    add("isize_one_short", p, b"twelve byte", INF_OUTPUT_OVERRUN, None)
    add("isize_one_long", p, b"twelve bytes!", INF_SIZE_MISMATCH, None)
    w = BitWriter()
    D.stored(w, b"abcdef", length=7)                                            # LEN one past the payload
    add("stored_past_the_payload", w.getvalue(), b"abcdefg", INF_INPUT_OVERRUN, "incomplete")
    # n literals: the end-of-block code (seven zero bits) takes bits 3..7 of byte n and two bits of byte n + 1, which is
    # cut.  A decoder may read the footer's first byte in its place: n is chosen so that its two low bits are zero too.
    n = next(k for k in range(8, 64) if zlib.crc32(b"A" * k) & 3 == 0)
    p = _fixed_payload([65] * n)
    assert len(p) == n + 2 and p[-1] == 0
    add("eob_past_the_payload", p[:-1], b"A" * n, INF_INPUT_OVERRUN, "incomplete")
    add("crc_flipped", _fixed_payload(tokens), bytes(tokens), INF_BAD_CRC, None,
        crc=zlib.crc32(bytes(tokens)) ^ (1 << 13))
    w = BitWriter()
    D.stored(w, b"stored bytes")
    add("crc_of_a_changed_stored_byte", w.getvalue().replace(b"stored", b"stores"), b"stores bytes", INF_BAD_CRC, None,
        crc=zlib.crc32(b"stored bytes"))
    return cases
