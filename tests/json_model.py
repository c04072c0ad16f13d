"""The classify step of csrc/ctmr_json.cu restated on Python ints, word for word: 64-byte blocks, the escaped characters
from odd backslash runs, the in-string mask as a prefix XOR of the unescaped quotes, both carries restarting at every
body start, and the carries between blocks as composed 2-bit -> 2-bit functions (an exclusive scan).  `byte_scan` is the
plain byte-at-a-time reading that the bit arithmetic must reproduce."""
from __future__ import annotations

M64 = (1 << 64) - 1
EVEN = 0x5555555555555555
IDENTITY = 0xE4  # state s -> s


def prefix_xor(x):
    for k in (1, 2, 4, 8, 16, 32):
        x ^= (x << k) & M64
    return x


def scan_block(bs, qt, S, state):
    """-> (escaped, in_string, state_out); state bit 0: the first byte is escaped, bit 1: inside a string"""
    esc, st = state & 1, state >> 1
    escd = instr = 0
    a, rest = 0, S
    while True:
        if (rest >> a) & 1:
            esc = st = 0
            rest &= ~(1 << a)
        b = (rest & -rest).bit_length() - 1 if rest else 64
        L = b - a
        seg = M64 if L == 64 else (1 << L) - 1
        B = (bs >> a) & seg & ~esc & M64
        follows = ((B << 1) | esc) & M64
        odd_starts = B & ~EVEN & ~follows & M64
        total = odd_starts + B
        s = total & M64
        e = (EVEN ^ ((s << 1) & M64)) & follows
        esc_next = (total >> 64) & 1 if L == 64 else (e >> L) & 1
        e &= seg
        Q = (qt >> a) & seg & ~e & M64
        x = (prefix_xor(Q) ^ (M64 if st else 0)) & seg
        st = (x >> (L - 1)) & 1
        esc = esc_next
        escd |= (e << a) & M64
        instr |= (x << a) & M64
        if b == 64:
            return escd, instr, esc | (st << 1)
        a = b


def compose(x, y):
    """block x, then block y"""
    r = 0
    for s in range(4):
        r |= ((y >> (2 * ((x >> (2 * s)) & 3))) & 3) << (2 * s)
    return r


def classify(text: bytes, starts):
    """-> (escaped, in_string) as lists of 64-bit words: pass 1 (tables), the exclusive scan, pass 2"""
    nblk = (len(text) + 63) // 64
    padded = text + b"\0" * (nblk * 64 - len(text))
    S = [0] * (nblk + 1)
    for o in starts:
        S[o >> 6] |= 1 << (o & 63)
    bs, qt = [0] * nblk, [0] * nblk
    for k in range(nblk):
        for i, c in enumerate(padded[64 * k:64 * k + 64]):
            if c == 0x5C:
                bs[k] |= 1 << i
            if c == 0x22:
                qt[k] |= 1 << i
    trans = []
    for k in range(nblk):
        t = 0
        for s in range(4):
            t |= scan_block(bs[k], qt[k], S[k], s)[2] << (2 * s)
        trans.append(t)
    carry, acc = [], IDENTITY
    for t in trans:
        carry.append(acc)
        acc = compose(acc, t)
    escd, instr = [], []
    for k in range(nblk):
        e, x, _ = scan_block(bs[k], qt[k], S[k], carry[k] & 3)
        escd.append(e)
        instr.append(x)
    return escd, instr


def byte_scan(text: bytes, starts):
    """the same masks read one byte at a time"""
    nblk = (len(text) + 63) // 64
    escd, instr = [0] * nblk, [0] * nblk
    sset = set(starts)
    esc = st = 0
    for i, c in enumerate(text):
        if i in sset:
            esc = st = 0
        bit = 1 << (i & 63)
        if esc:
            escd[i >> 6] |= bit
            esc = 0
            if st:
                instr[i >> 6] |= bit
            continue
        if c == 0x5C:
            esc = 1
        elif c == 0x22:
            st ^= 1
        if st or (c == 0x22 and st):
            instr[i >> 6] |= bit
    return escd, instr
