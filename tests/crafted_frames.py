"""The catalogue of hand-built frames (tests/frame_writer.py) that the decode tests run on every path.

`catalogue()` returns [Case]: name, frame bytes, expected content (None: every decoder must reject the frame), the trace
the executor predicts ([(ll, ml, offset)], sequences per compressed block) and the dictionary.  Everything comes from
fixed seeds.  Groups, in the order they were built:
  offsets and repcodes -- the entropy code at its limits -- execute-kernel dependencies -- table modes the reference
  encoder never writes -- headers and dictionaries.
"""
import numpy as np

from tests import frame_writer as fw
from tests.frame_writer import Comp, Dictionary, Frame, Lits, Raw, Rle, FSE, PRE, REP, RLE_T


class Case:
    """`note`, when set, names a frame that RFC 8878 makes invalid but the reference accepts: every path here rejects it."""

    def __init__(self, name, frame, expected, trace, dictionary=None, note="", size=None):
        self.name, self.frame, self.expected, self.trace, self.note = name, frame, expected, trace, note
        # the size the header declares: a decoder that wrongly accepts a malformed frame regenerates exactly this much,
        # so the size checks of the batch call cannot hide it
        self.size = len(expected) if expected is not None else size
        self.dict = dictionary.data if dictionary is not None else b""
        self.dict_obj = dictionary
        self.bitplans = []                      # per compressed block with sequences: see frame_writer.window_margins


def _text(rng, n):
    words = [b"alpha ", b"beta ", b"gamma ", b"delta ", b"epsilon ", b"zeta ", b"eta ", b"theta ", b"\n", b"1234 ", b"{\"k\": "]
    out = bytearray()
    while len(out) < n:
        out += words[int(rng.integers(0, len(words)))]
    return bytes(out[:n])


def _norm(rng, nsym, log, used, minus1=0, big=None):
    """Normalized counts over symbols 0..nsym-1 summing to 2^log: every symbol in `used` gets >= 1, `minus1` other
    symbols get -1, the rest of the mass is spread at random (or given to `big`)."""
    norm = [0] * nsym
    for s in used:
        norm[s] = 1
    others = [s for s in range(nsym) if s not in used]
    for s in rng.permutation(others)[:minus1]:
        norm[int(s)] = -1
    left = (1 << log) - sum(1 if c == -1 else c for c in norm)
    assert left >= 0
    pos = [s for s in range(nsym) if norm[s] > 0]
    if big is not None:
        norm[big] += left
    else:
        for _ in range(left):
            norm[pos[int(rng.integers(0, len(pos)))]] += 1
    while norm and norm[-1] == 0:
        norm.pop()
    return norm


def _random_block(rng, hist, size, max_off=None, reps=True, ll_max=20, ml_max=40):
    """(literals, seqs) regenerating about `size` bytes after `hist` bytes of history: literal runs 0..20, matches 3..40,
    offsets within the history, some repcodes."""
    seqs, lits, n = [], bytearray(), 0
    max_off = max_off or 1 << 30
    while n < size - 60:
        ll = int(rng.integers(0 if hist + n else 1, ll_max))
        ml = int(rng.integers(3, ml_max + 1))
        avail = hist + n + ll
        r = rng.random()
        if reps and r < 0.25 and seqs:
            ov = int(rng.integers(1, 3))            # rep0 / rep1 (LL 0: rep1 / rep2), always inside a valid history
        else:
            ov = int(rng.integers(1, min(avail, max_off) + 1)) + 3
        seqs.append((ll, ml, ov))
        lits += _text(rng, ll)
        n += ll + ml
    lits += _text(rng, max(0, size - n))
    return bytes(lits), seqs


def _valid_reps(seqs, hist, reps=(1, 4, 8)):
    """Drop the repcode sequences of `seqs` that would point outside the history (keeps random blocks valid)."""
    rep, out, n = list(reps), [], hist
    for ll, ml, ov in seqs:
        if ov > 3:
            off = ov - 3
            nrep = [off, rep[0], rep[1]]
        else:
            idx = ov - 1 + (ll == 0)
            off = [rep[0], rep[1], rep[2], rep[0] - 1][idx]
            nrep = rep if idx == 0 else ([off, rep[0], rep[2]] if idx == 1 else [off, rep[0], rep[1]])
        if off < 1 or off > n + ll:
            ov, off, nrep = n + ll + 3, n + ll, [n + ll, rep[0], rep[1]]
        out.append((ll, ml, ov))
        rep = nrep
        n += ll + ml
    return out


def _tables(rng, seqs, logs=(9, 8, 9), minus1=(0, 0, 0), extra=((), (), ())):
    """FSE tables (LL, OF, ML) at the given logs that hold every code of `seqs` (plus `extra` symbols)."""
    used = [sorted({fw.ll_code(a)[0] for a, _, _ in seqs} | set(extra[0])), sorted({fw.of_code(c)[0] for _, _, c in seqs} | set(extra[1])),
            sorted({fw.ml_code(b)[0] for _, b, _ in seqs} | set(extra[2]))]
    return [FSE(_norm(rng, n, lg, u, minus1=min(m, n - len(u))), lg) for n, lg, u, m in zip((36, 32, 53), logs, used, minus1)]


def _case(out, name, F, D=None, note=""):
    frame, expected, trace = fw.write(F, D)
    out.append(Case(name, frame, expected, trace, D, note, fw.regen_size(F)))
    out[-1].bitplans = [B.bitplan for B in F.blocks if isinstance(B, Comp) and B.seqs]


# --- group 1: offsets and repcodes -----------------------------------------------------------------------------------
def _offsets(out, rng):
    pre = _text(rng, 3000)
    for c in (29, 30, 31):
        for eb in (0, 3, min((1 << 31) - 1, (1 << c) - 1)):
            ov = (1 << c) + eb
            bad = Comp(Lits(b"q" * 20), [(4, 5, ov)], of=RLE_T(c))
            _case(out, "of%d_extra%d_first_block" % (c, eb), Frame([bad]))
            _case(out, "of%d_extra%d_after_raw" % (c, eb), Frame([Raw(pre), bad]))
            good = Comp(Lits(pre[:200]), [(10, 20, 4), (5, 9, 100)])
            _case(out, "of%d_extra%d_after_compressed" % (c, eb), Frame([good, Comp(Lits(b"q" * 20), [(4, 5, 7), (1, 5, ov)], of=FSE([0, 0, 16] + [0] * (c - 3) + [16], 5))]))
    # every repcode case at the first sequence of a block that follows a compressed block (symbolic on the block path)
    setup = Comp(Lits(pre[:600]), [(100, 10, 103), (100, 10, 203), (100, 10, 303)])      # reps 300, 200, 100
    for ll, ov, what in ((5, 1, "rep0"), (5, 2, "rep1"), (5, 3, "rep2"), (0, 1, "ll0_rep1"), (0, 2, "ll0_rep2"), (0, 3, "ll0_rep0_minus1")):
        follow = [(ll, 12, ov), (0, 7, 1), (3, 9, 1), (0, 5, 3), (2, 8, 3), (4, 6, 2)]
        _case(out, "repcode_%s_at_block_start" % what, Frame([setup, Comp(Lits(pre[600:650]), follow),
                                                              Comp(Lits(pre[650:700]), [(0, 11, 3), (6, 4, 2), (0, 4, 1)])]))
        _case(out, "repcode_%s_after_raw_block" % what, Frame([setup, Raw(pre[:77]), Comp(Lits(pre[600:650]), follow)]))
    # a chain of blocks that only use repcodes: the entry history of block k is the exit of k - 1, symbolic all the way
    chain = [setup] + [Comp(Lits(pre[k * 40:k * 40 + 40]), [(0, 5 + k, 1 + k % 3), (3, 4, 1 + (k + 1) % 3), (0, 6, 3)]) for k in range(8)]
    _case(out, "repcode_chain_over_9_blocks", Frame(chain))
    # rep0 - 1 == 0 as a block's last sequence, then another block
    for where in ("first", "later"):
        blocks = [] if where == "first" else [setup]
        blocks += [Comp(Lits(pre[:40]), [(10, 5, 40), (4, 6, 4), (0, 5, 3)]), Comp(Lits(pre[:40]), [(5, 5, 1), (0, 5, 2)])]
        _case(out, "rep0_minus1_is_zero_%s_block_then_another" % where, Frame(blocks))
        blocks[-1] = Comp(Lits(pre[:40]), [(5, 5, 50), (0, 5, 2)])
        _case(out, "rep0_minus1_is_zero_%s_block_then_new_offsets" % where, Frame(blocks))
    # rep0 - 1 from a symbolic history: the same chain with rep0 = 2 is valid (offset 1)
    _case(out, "rep0_minus1_to_offset_1", Frame([Comp(Lits(pre[:40]), [(10, 5, 5)]), Comp(Lits(pre[:40]), [(0, 5, 3), (3, 5, 1)])]))
    # dictionary repcodes used by the first sequence, reaching exactly to the start of the dictionary content
    content = _text(rng, 1500)
    wts = [0] * 10 + [1, 1, 2]
    D_tabs = dict(of=FSE(fw.OF_DEFAULT[0], 5), ml=FSE(fw.ML_DEFAULT[0], 6), ll=FSE(fw.LL_DEFAULT[0], 6))
    C = len(content)
    for reps, ll, ov, what in (((C, 5, 9), 4, 1, "rep0"), ((7, C, 9), 0, 1, "ll0_rep1"), ((7, 5, C), 0, 2, "ll0_rep2"),
                               ((9, C, 5), 3, 2, "rep1"), ((9, 5, C), 3, 3, "rep2"), ((C, 5, 9), 0, 3, "ll0_rep0_minus1")):
        D = Dictionary(content, dict_id=77, weights=wts, reps=reps, **D_tabs)
        _case(out, "dict_%s_reaches_content_start" % what, Frame([Comp(Lits(b"\x0a\x0b\x0c\x0a\x0b"), [(ll, 40, ov), (1, 30, 1)], ll=REP, of=REP, ml=REP)], dict_id=77), D)
    D = Dictionary(content, dict_id=78, weights=wts, reps=(C, 5, 9), **D_tabs)
    _case(out, "dict_offset_two_before_content_start", Frame([Comp(Lits(b"\x0a" * 8), [(0, 40, 4 + C + 1)])], dict_id=78), D,
          note="the history is the dictionary content (RFC 8878 section 5); the reference's DDict also keeps its header bytes")
    _case(out, "dict_new_offset_exactly_content_start", Frame([Comp(Lits(b"\x0a" * 8), [(3, 40, 3 + C + 3)])], dict_id=78), D)


# --- group 2: the entropy code at its limits -------------------------------------------------------------------------
def _entropy(out, rng):
    hist = _text(rng, 131072)
    big = Raw(hist)
    for k, (llog, olog, mlog, m1) in enumerate(((9, 8, 9, 0), (9, 8, 9, 12), (5, 5, 5, 0), (5, 5, 5, 3), (9, 8, 9, 30), (6, 7, 8, 5))):
        small = llog < 7
        lits, seqs = _random_block(rng, 131072, 30000 if small else 100000, max_off=130000, ll_max=16 if small else 20, ml_max=18 if small else 40)
        seqs = _valid_reps(seqs, 131072)
        codes = [(fw.ll_code(a)[0], fw.of_code(c)[0], fw.ml_code(b)[0]) for a, b, c in seqs]
        used = [sorted({x[i] for x in codes}) for i in range(3)]
        tl = FSE(_norm(rng, 36, llog, used[0] + [35], minus1=min(m1, 36 - len(used[0]) - 1)), llog) if len(used[0]) < 1 << llog else PRE
        to = FSE(_norm(rng, 32, olog, used[1], minus1=min(m1, 32 - len(used[1]))), olog)
        tm = FSE(_norm(rng, 53, mlog, used[2] + [52], minus1=min(m1, 53 - len(used[2]) - 1)), mlog)
        _case(out, "tables_logs_%d_%d_%d_minus1_%d" % (llog, olog, mlog, m1), Frame([big, Comp(Lits(lits), seqs, ll=tl, of=to, ml=tm)], window_log=18))
    # one symbol holds all 2^log states: the x = 1023 cells at log 9 (ML, LL), 511 at log 8 (OF)
    for llog, olog, mlog in ((9, 8, 9), (5, 5, 5), (9, 5, 6)):
        seqs = [(7, 20, 104)] * 40
        one = lambda sym, log: FSE([0] * sym + [1 << log], log)
        _case(out, "one_symbol_holds_every_state_%d_%d_%d" % (llog, olog, mlog),
              Frame([Raw(hist[:2000]), Comp(Lits(hist[:280]), seqs, ll=one(7, llog), of=one(6, olog), ml=one(17, mlog))]))
        _case(out, "one_symbol_holds_every_state_then_repeat_%d_%d_%d" % (llog, olog, mlog),
              Frame([Raw(hist[:2000]), Comp(Lits(hist[:280]), seqs, ll=one(7, llog), of=one(6, olog), ml=one(17, mlog)),
                     Comp(Lits(hist[:70]), seqs[:10], ll=REP, of=REP, ml=REP)]))
    # the largest codes: LL 35 and ML 52 (16 extra bits each), in blocks of their own
    _case(out, "ll_code_35", Frame([Comp(Lits(hist[:70000]), [(65536 + 4000, 30, 1000)], ll=FSE(_norm(rng, 36, 9, [35]), 9))], window_log=18))
    _case(out, "ml_code_52", Frame([Raw(hist[:5000]), Comp(Lits(hist[:10]), [(5, 65539 + 60000, 4000)], ml=_ml52(rng))], window_log=18))
    seqs = [(65536 + 100, 30, 4003), (3, 4000, 2), (10, 40000, 1)]
    tl, to, tm = _tables(rng, seqs, minus1=(5, 5, 5), extra=((35,), (), (52,)))
    _case(out, "ll_35_ml_52_in_one_table", Frame([Raw(hist[:5000]), Comp(Lits(hist[:70000]), seqs, ll=tl, of=to, ml=tm)], window_log=18))
    # every sequence takes the decoder's slow refill: 17 offset bits + 12 LL bits + 10 ML bits + 26 state bits > 64
    slow = [(4096 + int(rng.integers(0, 4096)), 1027 + int(rng.integers(0, 1024)), (1 << 17) + int(rng.integers(0, 1 << 17))) for _ in range(16)]
    lits = _text(rng, sum(s[0] for s in slow))
    ln = FSE(_norm(rng, 36, 9, [31], big=0), 9)
    on = FSE(_norm(rng, 32, 8, [17], big=0), 8)
    mn = FSE(_norm(rng, 53, 9, [46], big=0), 9)
    pre2 = _text(rng, 131072)
    _case(out, "slow_refill_every_sequence", Frame([Raw(hist), Raw(pre2), Comp(Lits(lits), slow, ll=ln, of=on, ml=mn)], window_log=20))
    # Sequences whose bits fill the decoder's window exactly (margin 0: no refill between the reads) or exceed it by one
    # (margin 1: the refill is needed), for every 16-byte alignment of the stream.  Blocks of widely varying bits per
    # sequence at the maximum logs are added until frame_writer.window_margins finds both margins at every alignment.
    need = {(skew, m) for skew in range(16) for m in (0, 1)}
    for k in range(40):
        if not need:
            break
        seqs, tot = [], 0
        while True:
            lc = int(rng.choice([0, 5, 17, 22, 24, 25]))
            mc = int(rng.choice([0, 9, 33, 38, 41, 43]))
            oc = int(rng.choice([2, 5, 9, 12, 14, 16]))
            s_ = (fw.LL_BASE[lc] + int(rng.integers(0, 1 << fw.LL_BITS[lc])), fw.ML_BASE[mc] + int(rng.integers(0, 1 << fw.ML_BITS[mc])),
                  (1 << oc) + int(rng.integers(0, 1 << oc)))
            if tot + s_[0] + s_[1] > 60000:
                break
            seqs.append(s_)
            tot += s_[0] + s_[1]
        tl, to, tm = _tables(rng, seqs, minus1=(6, 4, 9))
        F = Frame([Raw(hist), Comp(Lits(_text(rng, sum(x[0] for x in seqs))), seqs, ll=tl, of=to, ml=tm)], window_log=18)
        frame, expected, trace = fw.write(F)
        plan = F.blocks[1].bitplan
        got = {(skew, m) for skew in range(16) for m in (0, 1) if m in fw.window_margins(plan, skew)}
        if got & need:
            need -= got
            out.append(Case("window_boundary_%d" % k, frame, expected, trace, None, "", len(expected)))
            out[-1].bitplans = [plan]
    assert not need, sorted(need)


def _ml52(rng):
    return FSE(_norm(rng, 53, 9, [52]), 9)


def stream_cases(rng):
    """Sequence bit streams of 1, 2, 15, 16, 17 and 63 bytes at every 16-byte phase: k raw literals in front shift them."""
    out = []
    hist = _text(rng, 300)
    for nbytes in (1, 2, 15, 16, 17, 63):
        n = (8 * nbytes - 1) // 7                # OF code 7 (7 extra bits) per sequence, RLE tables: 7n + 1 bits
        for k in range(16):
            seqs = [(0, 3 + (i % 5), 128 + int(rng.integers(0, 128))) for i in range(n)]
            _case(out, "stream_%d_bytes_phase_%d" % (nbytes, k), Frame([Raw(hist), Comp(Lits(hist[:k]), seqs, ll=RLE_T(0), of=RLE_T(7), ml=PRE)]))
    return out


# --- group 3: execute-kernel dependencies ----------------------------------------------------------------------------
def _execute(out, rng):
    for size in (4095, 4096, 4097):
        for k in range(2):
            lits, seqs = _random_block(rng, 0, size, reps=True)
            seqs = _valid_reps(seqs, 0)
            regen = len(lits) + sum(s[1] for s in seqs)
            lits = lits + _text(rng, size - regen) if regen < size else lits
            if regen > size:                   # trim the last literals
                lits = lits[:len(lits) - (regen - size)]
            assert len(seqs) >= 64
            _case(out, "frame_%d_bytes_%d" % (size, k), Frame([Comp(Lits(lits, "raw"), seqs)]))
    # each match's source is the previous match or starts right at / just before its end: e == srcp at the frontier
    for delta in (0, 1, 2, "prev"):
        for total in (4000, 12000):
            seqs, n, prev_ml = [], 0, 0
            lits = bytearray()
            first = _text(rng, 50)
            while n < total - 100:
                ll = int(rng.integers(1, 4))
                ml = int(rng.integers(3, 41))
                if not seqs:
                    off = 7
                else:
                    off = ll + (prev_ml if delta == "prev" else delta) if delta != 0 else ll
                if delta == "prev" and ml > prev_ml:
                    ml = max(3, prev_ml)
                off = max(1, min(off, n + ll))
                seqs.append((ll, ml, off + 3))
                lits += first[len(lits) % 40:len(lits) % 40 + ll]
                n += ll + ml
                prev_ml = ml
            _case(out, "chained_sources_delta_%s_%d" % (delta, total), Frame([Comp(Lits(bytes(lits)), seqs)]))
    # short offsets 1..7 with lengths 3..40; long matches with o < 32 and o >= 32; a match ending at the frame's last byte
    seqs = [(1, ml, off + 3) for off in range(1, 8) for ml in (3, 4, 7, 8, 9, 16, 31, 32, 33, 40)]
    _case(out, "short_offsets", Frame([Comp(Lits(_text(rng, len(seqs))), seqs)]))
    seqs = [(2, 32 + k, (5 + 7 * k) + 3) for k in range(30)] + [(0, 200, 3 + 33), (0, 64, 3 + 31)]
    _case(out, "long_matches_near_and_far", Frame([Raw(_text(rng, 400)), Comp(Lits(_text(rng, 60)), seqs)]))
    _case(out, "match_ends_at_last_byte", Frame([Comp(Lits(b"0123456789"), [(10, 3000, 3 + 10)])]))
    # dictionary sources: matches of >= 32 bytes that start in the dictionary (o > position), and one that runs past its end
    content = _text(rng, 2000)
    D = Dictionary(content, raw=True)
    seqs = [(0, 40, 3 + 2000), (3, 33, 3 + 500), (1, 64, 3 + 1900), (0, 100, 3 + 150), (5, 50, 3 + 30)]
    _case(out, "raw_dict_long_matches", Frame([Comp(Lits(b"abcdefghi"), seqs)]), D)
    _case(out, "raw_dict_match_runs_into_frame", Frame([Comp(Lits(b"XYZW"), [(4, 300, 3 + 100)])]), D)
    _case(out, "raw_dict_offset_one_past", Frame([Comp(Lits(b"XYZW"), [(4, 30, 3 + 2005)])]), D)
    # block path: blocks of 6143, 6144, 6145 sequences (its per-block capacity), matches reaching several blocks back
    far = _text(rng, 40000)                     # sources in a raw block in front: no chains inside the long blocks
    for nseq in (6143, 6144, 6145):
        seqs = [(0, 3 + (i % 4), 3 + 30000 + 7 * (i % 500)) for i in range(nseq)]
        _case(out, "block_of_%d_sequences" % nseq, Frame([Raw(far), Comp(Lits(b""), seqs, ll=RLE_T(0), ml=PRE), Comp(Lits(b"e"), seqs[:100], ll=RLE_T(0))], window_log=18))
    blocks = [Raw(_text(rng, 20000))]
    for k in range(5):
        seqs = [(3, 30, 3 + 15000 + 9900 * k + 7 * i) for i in range(300)]      # each block regenerates 9900 bytes
        blocks.append(Comp(Lits(_text(rng, 900)), seqs))
    _case(out, "matches_reach_several_blocks_back", Frame(blocks, window_log=18))
    # offset-1 runs across whole 128 KiB blocks (the pointer-jumping executor's deepest chains)
    _case(out, "offset_1_run_whole_blocks", Frame([Comp(Lits(b"a"), [(1, 131071, 4)]), Comp(Lits(b"b"), [(1, 65539 + 60000, 4), (0, 5000, 1)]),
                                                   Comp(Lits(b""), [(0, 131072, 1)], ml=FSE(_norm(rng, 53, 6, [52]), 6))], window_log=18))


# --- group 4: table modes the reference encoder never writes ---------------------------------------------------------
def _modes(out, rng):
    t = _text(rng, 5000)
    s1 = [(30, 10, 30), (3, 8, 1), (0, 9, 2)]       # 33 literals
    s2 = [(4, 6, 1), (0, 7, 40), (2, 5, 2)]
    a = Comp(Lits(t[:30]), [(5, 10, 20), (5, 10, 30)], ll=RLE_T(5), of=RLE_T(4), ml=RLE_T(7))
    _case(out, "repeat_after_rle", Frame([Raw(t[:100]), a,
                                          Comp(Lits(t[:30]), [(5, 10, 25), (5, 10, 17)], ll=REP, of=REP, ml=REP)]))
    _case(out, "repeat_after_predefined", Frame([Comp(Lits(t[:40]), s1), Comp(Lits(t[:30]), s2, ll=REP, of=REP, ml=REP)]))
    _case(out, "repeat_across_raw_and_rle_blocks", Frame([Raw(t[:100]), a, Raw(t[:100]), Rle(0x41, 500), Comp(Lits(t[:40]), [(5, 10, 25), (5, 10, 16)], ll=REP, of=REP, ml=REP)]))
    _case(out, "repeat_across_empty_sequence_block", Frame([Raw(t[:100]), a, Comp(Lits(t[:20])), Comp(Lits(t[:40]), [(5, 10, 24), (5, 10, 19)], ll=REP, of=REP, ml=REP)]))
    _case(out, "repeat_in_first_block_without_dict", Frame([Comp(Lits(t[:40]), s1, ll=REP)]))
    _case(out, "repeat_of_only_in_first_block_without_dict", Frame([Comp(Lits(t[:40]), s1, of=REP)]))
    wts = [0] * 48 + [2, 2, 1, 1, 1, 1]             # '0'..'5'
    digits = bytes(48 + int(x) for x in rng.integers(0, 6, 3000))
    _case(out, "treeless_in_first_block_without_dict", Frame([Comp(Lits(digits[:300], "treeless", weights=wts), s1)]))
    content = _text(rng, 1000)
    D = Dictionary(content, dict_id=5, weights=wts, reps=(1, 4, 8), of=FSE(_norm(rng, 32, 8, list(range(12))), 8),
                   ml=FSE(_norm(rng, 53, 9, list(range(30))), 9), ll=FSE(_norm(rng, 36, 9, list(range(16))), 9))
    _case(out, "treeless_and_repeat_in_first_block_with_dict", Frame([Comp(Lits(digits[:300], "treeless"), [(5, 10, 30), (3, 8, 1), (0, 9, 2)], ll=REP, of=REP, ml=REP)], dict_id=5), D)
    _case(out, "repeat_in_first_block_with_dict_then_new", Frame([Comp(Lits(digits[:300], "treeless", streams=1), [(4, 9, 35), (0, 9, 2)], ll=REP, of=REP, ml=REP),
                                                                  Comp(Lits(digits[:300], "huf", weights=[0] * 48 + [1, 1, 2, 3, 3, 3]), [(5, 10, 14)])], dict_id=5), D)
    # a Huffman table of log 12
    w12 = [12, 11, 10, 9, 8, 7, 6, 5, 4, 3, 2, 1, 1]
    skew = bytes(int(min(12, x)) for x in rng.geometric(0.5, 2000) - 1)
    for streams in (1, 4):
        _case(out, "huffman_log_12_%d_streams" % streams, Frame([Comp(Lits(skew[:900], "huf", weights=w12, streams=streams), [(10, 20, 13)])]))
    _case(out, "huffman_log_12_fse_weights", Frame([Comp(Lits(skew[:2000], "huf", weights=w12, weights_fse=([0, 9, 3, 3, 3, 2, 2, 2, 2, 2, 2, 1, 1], 5)), [(10, 20, 13)])]))
    # 4 streams with 1..12 literals (fewer than 6 is malformed), and the empty 4th stream
    for regen in range(1, 13):
        _case(out, "four_streams_%d_literals" % regen, Frame([Comp(Lits(digits[:regen], "huf", weights=wts, streams=4), [(1, 4, 4)] if regen else [])]))
    # a 1-stream table reused as treeless with 4 streams; treeless after treeless; a new table after treeless
    _case(out, "one_stream_table_reused_by_four", Frame([Comp(Lits(digits[:200], "huf", weights=wts, streams=1), [(5, 6, 7)]),
                                                        Comp(Lits(digits[200:700], "treeless", streams=4), [(5, 6, 7)]),
                                                        Comp(Lits(digits[700:720], "treeless", streams=1), [(5, 6, 7)]),
                                                        Raw(t[:10]),
                                                        Comp(Lits(digits[:600], "treeless", streams=4, hdr=5))]))
    # sequence counts at the edges of the 1-, 2- and 3-byte forms
    _case(out, "zero_sequences", Frame([Comp(Lits(t[:100]))]))
    _case(out, "zero_sequences_with_trailing_bytes", Frame([Comp(Lits(t[:100]), trailing=b"\x00")]))
    _case(out, "count_5_in_two_byte_form", Frame([Comp(Lits(t[:100]), s1 + s2[:2], nseq_bytes=2)]))
    far = _text(rng, 131072)
    for n in (127, 128, 32511, 32512, 32513):
        seqs = [(0, 3, 3 + 100000 + 3 * (i % 1000)) for i in range(n)]
        _case(out, "sequence_count_%d" % n, Frame([Raw(far), Comp(Lits(b""), seqs, ll=RLE_T(0), of=PRE, ml=RLE_T(0))], window_log=18))
    # raw / RLE literal headers in all three sizes
    for hdr in (1, 2, 3):
        s3 = [(10, 10, 12), (3, 8, 1), (0, 9, 2)]      # 13 literals: fits the 5-bit size of the 1-byte header
        _case(out, "raw_literals_header_%d" % hdr, Frame([Comp(Lits(t[:20], "raw", hdr=hdr), s3)]))
        _case(out, "rle_literals_header_%d" % hdr, Frame([Comp(Lits(b"z", "rle", hdr=hdr, regen=25), s3)]))
    for hdr in (3, 4, 5):
        _case(out, "huffman_literals_header_%d" % hdr, Frame([Comp(Lits(digits[:900], "huf", weights=wts, streams=4, hdr=hdr), s1)]))


# --- group 5: headers and dictionaries -------------------------------------------------------------------------------
def _headers(out, rng):
    t = _text(rng, 70000)
    s1 = [(30, 10, 30), (3, 8, 1)]                 # 33 literals, 18 match bytes
    for size, fcs in ((100, 1), (100, 4), (100, 8), (300, 2), (65791, 2), (65792, 4), (3000, 8)):
        for single in (True, False):
            if fcs == 1 and not single:
                continue
            blocks = [Comp(Lits(t[:size - 18]), s1)] if size < 60000 else [Raw(t[:size - 51 - 60000]), Raw(t[:60000]), Comp(Lits(t[:33]), s1)]
            _case(out, "fcs_%d_bytes_size_%d_%s" % (fcs, size, "single" if single else "window"), Frame(blocks, single_segment=single, fcs_bytes=fcs, window_log=17))
    _case(out, "no_content_size", Frame([Comp(Lits(t[:40]), s1)], content_size=False))
    _case(out, "wrong_content_size", Frame([Comp(Lits(t[:40]), s1)], content_size=59))
    _case(out, "checksum", Frame([Comp(Lits(t[:4000]), s1)], checksum=True))
    _case(out, "wrong_checksum", Frame([Comp(Lits(t[:4000]), s1)], checksum=True, bad_checksum=True))
    _case(out, "window_mantissa_7", Frame([Raw(t[:1500]), Comp(Lits(t[:300]), s1)], window_log=10, window_mantissa=7))
    lenient = "RFC 8878 caps every block at min(window, 128 KiB); the reference checks only compressed blocks"
    _case(out, "raw_block_larger_than_window", Frame([Raw(t[:1500])], window_log=10), note=lenient)
    _case(out, "rle_block_larger_than_window", Frame([Rle(7, 1100)], window_log=10), note=lenient)
    _case(out, "compressed_block_larger_than_window", Frame([Comp(Lits(t[:1200]), s1)], window_log=10))
    _case(out, "raw_block_larger_than_128k", Frame([Raw(t[:65536] + t[:65537])], window_log=20), note=lenient)
    _case(out, "skippable_frame_in_front", Frame([Comp(Lits(t[:40]), s1)], skippable=b"skip me" * 3))
    wts = [0] * 32 + [1, 1] + [0] * 63 + [4, 3, 3, 2, 2, 2, 2, 2, 1, 1, 1, 1]
    content = _text(rng, 3000)
    D99 = Dictionary(content, dict_id=0x01020304, weights=wts, reps=(3000, 2999, 1),
                     of=FSE(_norm(rng, 32, 8, [0, 1, 2, 3, 4, 5, 8, 9, 10, 11, 12], minus1=5), 8),
                     ml=FSE(_norm(rng, 53, 9, list(range(0, 40)) + [52], minus1=10), 9),
                     ll=FSE(_norm(rng, 36, 9, list(range(0, 20)) + [35], minus1=4), 9))
    body = bytes(int(x) for x in rng.choice([32, 33] + list(range(97, 109)), 400))
    for did, dib in ((0x01020304, 4), (0x01020304, 0)):
        _case(out, "dict_tables_9_8_9_id_bytes_%d" % dib, Frame([Comp(Lits(body, "treeless"), [(10, 40, 1), (0, 33, 2), (3, 20, 3), (7, 8, 3000 + 3 + 7 + 40 + 33 + 3 + 20)], ll=REP, of=REP, ml=REP),
                                                             Comp(Lits(body[:100], "treeless"), [(10, 40, 1)], ll=REP, of=REP, ml=REP)],
                                                            dict_id=did, dict_id_bytes=dib), D99)
    for did, dib in ((200, 1), (40000, 2), (0xFFFFFF01, 4)):
        D = Dictionary(content, dict_id=did, weights=wts, reps=(1, 4, 8), of=FSE(fw.OF_DEFAULT[0], 5), ml=FSE(fw.ML_DEFAULT[0], 6), ll=FSE(fw.LL_DEFAULT[0], 6))
        _case(out, "dict_id_%d_bytes" % dib, Frame([Comp(Lits(body[:50], "treeless"), [(3, 50, 1000 + 3)])], dict_id=did, dict_id_bytes=dib), D)
    D = Dictionary(content, dict_id=9, weights=wts, reps=(1, 4, 8), of=FSE(fw.OF_DEFAULT[0], 5), ml=FSE(fw.ML_DEFAULT[0], 6), ll=FSE(fw.LL_DEFAULT[0], 6))
    _case(out, "dict_id_mismatch", Frame([Comp(Lits(body[:50], "treeless"), [(3, 50, 1000 + 3)])], dict_id=10), D)
    _case(out, "dict_huffman_weights_fse", Frame([Comp(Lits(body[:300], "treeless"), [(3, 50, 1000 + 3)])], dict_id=11),
          Dictionary(content, dict_id=11, weights=wts, weights_fse=([12, 8, 6, 4, 2], 5), reps=(3000, 1, 2),
                     of=FSE(fw.OF_DEFAULT[0], 5), ml=FSE(fw.ML_DEFAULT[0], 6), ll=FSE(fw.LL_DEFAULT[0], 6)))


def dict_rep_cases(rng):
    """Dictionaries whose repcodes equal the content size (valid) and exceed it by one (rejected when loaded)."""
    content = _text(rng, 800)
    tabs = dict(of=FSE(fw.OF_DEFAULT[0], 5), ml=FSE(fw.ML_DEFAULT[0], 6), ll=FSE(fw.LL_DEFAULT[0], 6))
    out = []
    for extra in (0, 1):
        for k in range(3):
            reps = [1, 4, 8]
            reps[k] = len(content) + extra
            D = Dictionary(content, dict_id=21, weights=[0] * 97 + [1, 1, 2], reps=reps, **tabs)
            _case(out, "dict_rep%d_content_size_plus_%d" % (k, extra), Frame([Comp(Lits(b"abcabc"), [(0, 20, [1, 1, 2][k]), (3, 5, 1)])], dict_id=21), D)
    return out


def catalogue():
    out = []
    _offsets(out, np.random.default_rng(101))
    _entropy(out, np.random.default_rng(102))
    _execute(out, np.random.default_rng(103))
    _modes(out, np.random.default_rng(104))
    _headers(out, np.random.default_rng(105))
    return out
