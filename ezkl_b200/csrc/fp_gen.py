#!/usr/bin/env python
"""Generates fp_ptx.cuh: inline-PTX 256-bit Montgomery arithmetic for BN254 Fr and Fq (8 x 32-bit limbs).

Why a generator: the carry chains (mad.lo.cc / madc.hi.cc ...) must live in ONE asm block per operation so the
compiler cannot disturb the CC flag, and there is no GPU in the build container.  The generator therefore also
contains a tiny PTX interpreter: every emitted instruction list is executed on random and edge-case inputs and
compared with Python bigint arithmetic BEFORE the header is written (``python fp_gen.py --check`` only checks).

Multiplication = operand-scanning Montgomery (CIOS) with the even/odd split accumulator: products a[j]*b_i for even
j tile limbs (0,1),(2,3).. and for odd j tile (1,2),(3,4).., so each row is two independent chains of
(lo,hi) pairs that ptxas can fuse into IMAD.WIDE.U32(.X) on sm_90a.  Modulus limbs are literal immediates.
"""
import random
import sys

M32 = 0xFFFFFFFF
FIELDS = {
    "fr": 0x30644e72e131a029b85045b68181585d2833e84879b9709143e1f593f0000001,
    "fq": 0x30644e72e131a029b85045b68181585d97816a916871ca8d3c208c16d87cfd47,
}


def limbs(x, n=8):
    return [(x >> (32 * i)) & M32 for i in range(n)]


# ---- instruction list builders -------------------------------------------------------------------------
def gen_mul(mod):
    """out[0..7] = a*b*2^-256 mod M, fully reduced.  Registers: a0..a7, b0..b7 in; r0..r7 out."""
    Ml = limbs(mod)
    inv = (-pow(mod, -1, 1 << 32)) & M32
    ins = []
    X = ["x%d" % i for i in range(8)]
    Y = ["y%d" % i for i in range(8)]
    A = ["a%d" % i for i in range(8)]
    B = ["b%d" % i for i in range(8)]

    def imm(v):
        return "0x%08x" % v

    def reduce_row(E, O):
        ins.append(("mul.lo.u32", "m", E[0], imm(inv)))
        for j in range(4):   # odd modulus limbs into O
            ins.append((("mad.lo.cc.u32" if j == 0 else "madc.lo.cc.u32"), O[2 * j], "m", imm(Ml[2 * j + 1]), O[2 * j]))
            ins.append(("madc.hi.cc.u32", O[2 * j + 1], "m", imm(Ml[2 * j + 1]), O[2 * j + 1]))
        for j in range(4):   # even modulus limbs into E
            ins.append((("mad.lo.cc.u32" if j == 0 else "madc.lo.cc.u32"), E[2 * j], "m", imm(Ml[2 * j]), E[2 * j]))
            ins.append(("madc.hi.cc.u32", E[2 * j + 1], "m", imm(Ml[2 * j]), E[2 * j + 1]))
        ins.append(("addc.u32", O[7], O[7], "0"))

    # row 0: plain products
    for j in range(4):
        ins.append(("mul.lo.u32", X[2 * j], A[2 * j], B[0]))
        ins.append(("mul.hi.u32", X[2 * j + 1], A[2 * j], B[0]))
    for j in range(4):
        ins.append(("mul.lo.u32", Y[2 * j], A[2 * j + 1], B[0]))
        ins.append(("mul.hi.u32", Y[2 * j + 1], A[2 * j + 1], B[0]))
    E, O = X, Y
    reduce_row(E, O)
    for i in range(1, 8):
        nE, nO = O, E      # shift by one limb: old O is even-aligned in the new frame, old E (>>2 limbs) is odd-aligned
        ins.append(("add.cc.u32", nE[0], nE[0], nO[1]))
        for j in range(4):
            c_lo = nO[2 * j + 2] if 2 * j + 2 < 8 else "0"
            c_hi = nO[2 * j + 3] if 2 * j + 3 < 8 else "0"
            ins.append(("madc.lo.cc.u32", nO[2 * j], A[2 * j + 1], B[i], c_lo))
            ins.append(("madc.hi.cc.u32", nO[2 * j + 1], A[2 * j + 1], B[i], c_hi))
        for j in range(4):
            ins.append((("mad.lo.cc.u32" if j == 0 else "madc.lo.cc.u32"), nE[2 * j], A[2 * j], B[i], nE[2 * j]))
            ins.append(("madc.hi.cc.u32", nE[2 * j + 1], A[2 * j], B[i], nE[2 * j + 1]))
        ins.append(("addc.u32", nO[7], nO[7], "0"))
        E, O = nE, nO
        reduce_row(E, O)
    # merge: t = (E >> 32) + O
    T = ["t%d" % i for i in range(8)]
    for j in range(7):
        ins.append((("add.cc.u32" if j == 0 else "addc.cc.u32"), T[j], O[j], E[j + 1]))
    ins.append(("addc.u32", T[7], O[7], "0"))
    ins += final_sub(T, Ml)
    return ins


def gen_mul2(mod):
    """out = (a*b + c*d) * 2^-256 mod M, fully reduced: ONE interleaved Montgomery reduction for two products.

    Row i adds a*b_i and c*d_i to the even/odd accumulator pair, then one reduction row.  With a, c <= M and the running
    value V_i < 3M(1 + 2^-32):  V_{i+1} = (V_i + a*b_i + c*d_i + m*M) / 2^32 < V_i / 2^32 + 3M, so the invariant holds and the
    value before each division stays below 3M*2^32 + 3M < 2^288 (M < 0.19 * 2^256): neither accumulator chain can carry out
    of its top limb except E into O[7], which every E chain is followed by.  The final value is exact:
    (a*b + c*d + m*M) / 2^256 with m < 2^256, i.e. < 2*M^2/2^256 + M < 1.4 M, so one conditional subtraction finishes."""
    Ml = limbs(mod)
    inv = (-pow(mod, -1, 1 << 32)) & M32
    ins = []
    X = ["x%d" % i for i in range(8)]
    Y = ["y%d" % i for i in range(8)]
    A = ["a%d" % i for i in range(8)]
    B = ["b%d" % i for i in range(8)]
    Cc = ["c%d" % i for i in range(8)]
    D = ["d%d" % i for i in range(8)]

    def imm(v):
        return "0x%08x" % v

    def acc_rows(E, O, P, q):
        """E/O += P * q (plain accumulate: odd limbs of P into O, even limbs into E, E's carry into O[7])."""
        def pair(p):                       # register operand first, immediate (modulus limb) second
            return (q, p) if p.startswith("0x") else (p, q)
        for j in range(4):
            ins.append((("mad.lo.cc.u32" if j == 0 else "madc.lo.cc.u32"), O[2 * j]) + pair(P[2 * j + 1]) + (O[2 * j],))
            ins.append(("madc.hi.cc.u32", O[2 * j + 1]) + pair(P[2 * j + 1]) + (O[2 * j + 1],))
        for j in range(4):
            ins.append((("mad.lo.cc.u32" if j == 0 else "madc.lo.cc.u32"), E[2 * j]) + pair(P[2 * j]) + (E[2 * j],))
            ins.append(("madc.hi.cc.u32", E[2 * j + 1]) + pair(P[2 * j]) + (E[2 * j + 1],))
        ins.append(("addc.u32", O[7], O[7], "0"))

    def reduce_row(E, O):
        ins.append(("mul.lo.u32", "m", E[0], imm(inv)))
        acc_rows(E, O, [imm(v) for v in Ml], "m")

    for j in range(4):
        ins.append(("mul.lo.u32", X[2 * j], A[2 * j], B[0]))
        ins.append(("mul.hi.u32", X[2 * j + 1], A[2 * j], B[0]))
    for j in range(4):
        ins.append(("mul.lo.u32", Y[2 * j], A[2 * j + 1], B[0]))
        ins.append(("mul.hi.u32", Y[2 * j + 1], A[2 * j + 1], B[0]))
    E, O = X, Y
    acc_rows(E, O, Cc, D[0])
    reduce_row(E, O)
    for i in range(1, 8):
        nE, nO = O, E
        ins.append(("add.cc.u32", nE[0], nE[0], nO[1]))
        for j in range(4):
            c_lo = nO[2 * j + 2] if 2 * j + 2 < 8 else "0"
            c_hi = nO[2 * j + 3] if 2 * j + 3 < 8 else "0"
            ins.append(("madc.lo.cc.u32", nO[2 * j], A[2 * j + 1], B[i], c_lo))
            ins.append(("madc.hi.cc.u32", nO[2 * j + 1], A[2 * j + 1], B[i], c_hi))
        for j in range(4):
            ins.append((("mad.lo.cc.u32" if j == 0 else "madc.lo.cc.u32"), nE[2 * j], A[2 * j], B[i], nE[2 * j]))
            ins.append(("madc.hi.cc.u32", nE[2 * j + 1], A[2 * j], B[i], nE[2 * j + 1]))
        ins.append(("addc.u32", nO[7], nO[7], "0"))
        E, O = nE, nO
        acc_rows(E, O, Cc, D[i])
        reduce_row(E, O)
    T = ["t%d" % i for i in range(8)]
    for j in range(7):
        ins.append((("add.cc.u32" if j == 0 else "addc.cc.u32"), T[j], O[j], E[j + 1]))
    ins.append(("addc.u32", T[7], O[7], "0"))
    ins += final_sub(T, Ml)
    return ins


def gen_sqr(mod):
    """out = a*a * 2^-256 mod M with 36 limb products instead of 64.

    a^2 = sum_i a_i 2^(32i) * (a_i 2^(32i) + 2 * sum_{j>i} a_j 2^(32j)).  With u = 2a (fits 8 limbs, a <= M < 2^254) and
    w_j = (2 a_j) mod 2^32, the bracket's limbs from position i up are exactly  [a_i, w_(i+1), u_(i+2), ..., u_7]  (u_(i+1)
    carries the top bit of a_i in its lowest bit; that bit belongs to the doubled a_i term, which is not wanted, so position
    i+1 uses w).  Row i of the interleaved reduction therefore multiplies only positions >= i by a_i; skipped odd positions
    still perform the one-limb shift of the accumulator (plain add-with-carry), skipped even positions need nothing.
    The running value stays below 3M(1 + 2^-32) as in gen_mul2 (each row adds < 2M * 2^32); the final value is
    (a^2 + m*M) / 2^256 < 2M."""
    Ml = limbs(mod)
    inv = (-pow(mod, -1, 1 << 32)) & M32
    ins = []
    X = ["x%d" % i for i in range(8)]
    Y = ["y%d" % i for i in range(8)]
    A = ["a%d" % i for i in range(8)]
    U = ["u%d" % i for i in range(8)]
    Wl = ["w%d" % i for i in range(8)]

    def imm(v):
        return "0x%08x" % v

    for j in range(1, 8):
        ins.append(("shl.b32", Wl[j], A[j], "1"))
    for j in range(2, 8):
        ins.append(("shf.l.clamp.b32", U[j], A[j - 1], A[j], "1"))

    def operand(i, j):                   # limb at position j of row i's multiplicand (j >= i)
        return A[j] if j == i else (Wl[j] if j == i + 1 else U[j])

    def reduce_row(E, O):
        ins.append(("mul.lo.u32", "m", E[0], imm(inv)))
        for j in range(4):
            ins.append((("mad.lo.cc.u32" if j == 0 else "madc.lo.cc.u32"), O[2 * j], "m", imm(Ml[2 * j + 1]), O[2 * j]))
            ins.append(("madc.hi.cc.u32", O[2 * j + 1], "m", imm(Ml[2 * j + 1]), O[2 * j + 1]))
        for j in range(4):
            ins.append((("mad.lo.cc.u32" if j == 0 else "madc.lo.cc.u32"), E[2 * j], "m", imm(Ml[2 * j]), E[2 * j]))
            ins.append(("madc.hi.cc.u32", E[2 * j + 1], "m", imm(Ml[2 * j]), E[2 * j + 1]))
        ins.append(("addc.u32", O[7], O[7], "0"))

    for j in range(4):
        ins.append(("mul.lo.u32", X[2 * j], operand(0, 2 * j), A[0]))
        ins.append(("mul.hi.u32", X[2 * j + 1], operand(0, 2 * j), A[0]))
    for j in range(4):
        ins.append(("mul.lo.u32", Y[2 * j], operand(0, 2 * j + 1), A[0]))
        ins.append(("mul.hi.u32", Y[2 * j + 1], operand(0, 2 * j + 1), A[0]))
    E, O = X, Y
    reduce_row(E, O)
    for i in range(1, 8):
        nE, nO = O, E
        ins.append(("add.cc.u32", nE[0], nE[0], nO[1]))
        for j in range(4):               # odd positions: product (if position >= i) fused with the shift, else the shift alone
            c_lo = nO[2 * j + 2] if 2 * j + 2 < 8 else "0"
            c_hi = nO[2 * j + 3] if 2 * j + 3 < 8 else "0"
            if 2 * j + 1 >= i:
                ins.append(("madc.lo.cc.u32", nO[2 * j], operand(i, 2 * j + 1), A[i], c_lo))
                ins.append(("madc.hi.cc.u32", nO[2 * j + 1], operand(i, 2 * j + 1), A[i], c_hi))
            else:
                ins.append(("addc.cc.u32", nO[2 * j], c_lo, "0"))
                ins.append(("addc.cc.u32", nO[2 * j + 1], c_hi, "0"))
        first = True
        for j in range(4):               # even positions >= i
            if 2 * j < i:
                continue
            ins.append((("mad.lo.cc.u32" if first else "madc.lo.cc.u32"), nE[2 * j], operand(i, 2 * j), A[i], nE[2 * j]))
            ins.append(("madc.hi.cc.u32", nE[2 * j + 1], operand(i, 2 * j), A[i], nE[2 * j + 1]))
            first = False
        if not first:
            ins.append(("addc.u32", nO[7], nO[7], "0"))
        E, O = nE, nO
        reduce_row(E, O)
    T = ["t%d" % i for i in range(8)]
    for j in range(7):
        ins.append((("add.cc.u32" if j == 0 else "addc.cc.u32"), T[j], O[j], E[j + 1]))
    ins.append(("addc.u32", T[7], O[7], "0"))
    ins += final_sub(T, Ml)
    return ins


def final_sub(T, Ml, out=None):
    """out = T - M if T >= M else T  (M given as limbs; out defaults to r0..r7)."""
    out = out or ["r%d" % i for i in range(8)]
    ins = []
    S = ["s%d" % i for i in range(8)]
    for j in range(8):
        ins.append((("sub.cc.u32" if j == 0 else "subc.cc.u32"), S[j], T[j], "0x%08x" % Ml[j]))
    ins.append(("subc.u32", "brw", "0", "0"))
    ins.append(("setp.eq.u32", "p", "brw", "0"))
    for j in range(8):
        ins.append(("selp.u32", out[j], S[j], T[j], "p"))
    return ins


def gen_add(mod):
    Ml = limbs(mod)
    ins = []
    T = ["t%d" % i for i in range(8)]
    for j in range(8):
        op = "add.cc.u32" if j == 0 else ("addc.cc.u32" if j < 7 else "addc.u32")
        ins.append((op, T[j], "a%d" % j, "b%d" % j))
    return ins + final_sub(T, Ml)


def gen_sub(mod):
    """r = a - b (+ M if borrow)."""
    Ml = limbs(mod)
    ins = []
    T = ["t%d" % i for i in range(8)]
    for j in range(8):
        ins.append((("sub.cc.u32" if j == 0 else "subc.cc.u32"), T[j], "a%d" % j, "b%d" % j))
    ins.append(("subc.u32", "brw", "0", "0"))       # 0xffffffff if a < b
    for j in range(8):
        ins.append(("and.b32", "s%d" % j, "brw", "0x%08x" % Ml[j]))
    for j in range(8):
        op = "add.cc.u32" if j == 0 else ("addc.cc.u32" if j < 7 else "addc.u32")
        ins.append((op, "r%d" % j, T[j], "s%d" % j))
    return ins


# ---- interpreter ---------------------------------------------------------------------------------------
def run(ins, regs):
    cc = 0
    pred = {}

    def val(x):
        if x in regs:
            return regs[x]
        return int(x, 0)

    for it in ins:
        op, d = it[0], it[1]
        s = [val(x) if x not in pred else x for x in it[2:]]
        if op == "mul.lo.u32":
            regs[d] = (s[0] * s[1]) & M32
        elif op == "mul.hi.u32":
            regs[d] = (s[0] * s[1]) >> 32
        elif op in ("mad.lo.cc.u32", "madc.lo.cc.u32", "madc.hi.cc.u32", "mad.hi.cc.u32"):
            p = s[0] * s[1]
            p = (p & M32) if ".lo" in op else (p >> 32)
            t = p + s[2] + (cc if op.startswith("madc") else 0)
            regs[d], cc = t & M32, t >> 32
        elif op in ("add.cc.u32", "addc.cc.u32", "addc.u32"):
            t = s[0] + s[1] + (cc if op.startswith("addc") else 0)
            regs[d] = t & M32
            if ".cc" in op:
                cc = t >> 32
        elif op in ("sub.cc.u32", "subc.cc.u32", "subc.u32"):
            t = s[0] - s[1] - (cc if op.startswith("subc") else 0)
            regs[d] = t & M32
            if ".cc" in op:
                cc = 1 if t < 0 else 0
        elif op == "and.b32":
            regs[d] = s[0] & s[1]
        elif op == "shl.b32":
            regs[d] = (s[0] << s[1]) & M32
        elif op == "shf.l.clamp.b32":          # upper word of ((hi:lo) << n), n <= 32
            regs[d] = ((((s[1] << 32) | s[0]) << min(s[2], 32)) >> 32) & M32
        elif op == "setp.eq.u32":
            pred[d] = (s[0] == s[1])
        elif op == "selp.u32":
            regs[d] = s[0] if pred[it[4]] else s[1]
        else:
            raise ValueError(op)
        assert 0 <= regs.get(d, 0) <= M32
    return regs


def check(name, mod, trials=3000):
    rng = random.Random(hash(name) & 0xFFFF)
    mul, add, sub = gen_mul(mod), gen_add(mod), gen_sub(mod)
    Rinv = pow(1 << 256, -1, mod)
    edge = [0, 1, 2, mod - 1, mod - 2, (1 << 254) % mod, (1 << 253), mod >> 1, 0xFFFFFFFF, (1 << 128) - 1]
    pairs = [(x, y) for x in edge for y in edge] + [(rng.randrange(mod), rng.randrange(mod)) for _ in range(trials)]
    for a, b in pairs:
        regs = {}
        for i, v in enumerate(limbs(a)):
            regs["a%d" % i] = v
        for i, v in enumerate(limbs(b)):
            regs["b%d" % i] = v
        for ins, exp in ((mul, a * b * Rinv % mod), (add, (a + b) % mod), (sub, (a - b) % mod)):
            out = run(ins, dict(regs))
            got = sum(out["r%d" % i] << (32 * i) for i in range(8))
            assert got == exp, (name, hex(a), hex(b), hex(got), hex(exp))
    # two-product multiply: operands up to and including M (a negated zero may arrive unreduced in principle)
    mul2 = gen_mul2(mod)
    edge2 = [0, 1, mod - 1, mod, (1 << 254) % mod, 0xFFFFFFFF, mod >> 1]
    quads = [(a, b, c, d) for a in edge2 for b in edge2 for c in edge2 for d in edge2]
    quads += [tuple(rng.randrange(mod) for _ in range(4)) for _ in range(trials)]
    for a, b, c, d in quads:
        regs = {}
        for nm, v in (("a", a), ("b", b), ("c", c), ("d", d)):
            for i, w in enumerate(limbs(v)):
                regs["%s%d" % (nm, i)] = w
        out = run(mul2, regs)
        got = sum(out["r%d" % i] << (32 * i) for i in range(8))
        exp = (a * b + c * d) * Rinv % mod
        assert got == exp, (name, "mul2", hex(a), hex(b), hex(c), hex(d), hex(got), hex(exp))
    sqr = gen_sqr(mod)
    for a in edge + [mod, (1 << 254) - 1 if (1 << 254) - 1 < mod else mod - 3, 0x80000000, 0xFFFFFFFF << 32, int("80000000" * 8, 16) % mod,
                     int("ffffffff" * 7, 16)] + [rng.randrange(mod) for _ in range(trials)]:
        regs = {"a%d" % i: v for i, v in enumerate(limbs(a))}
        out = run(sqr, regs)
        got = sum(out["r%d" % i] << (32 * i) for i in range(8))
        assert got == a * a * Rinv % mod, (name, "sqr", hex(a), hex(got))
    return len(mul), len(add), len(sub), len(mul2), len(sqr)


# ---- emitter -------------------------------------------------------------------------------------------
def emit_fn(fname, ins, n_in):
    """One asm block; outputs %0..%7 = r, inputs a = %8..%15, b = %16..%23 (if n_in == 2)."""
    tmp = sorted({x for it in ins for x in it[1:] if x[0] in "xytsmuw" and not x.startswith("0x")} | {"brw"})
    tmp = [t for t in tmp if t != "p"]
    lines = ["    .reg .u32 %s;" % ", ".join(tmp), "    .reg .pred p;"]

    def opnd(x):
        if x[0] == "r" and x[1:].isdigit():
            return "%%%d" % int(x[1:])
        if x[0] == "a" and x[1:].isdigit():
            return "%%%d" % (8 + int(x[1:]))
        if x[0] == "b" and x[1:].isdigit() and x != "brw":
            return "%%%d" % (16 + int(x[1:]))
        if x[0] == "c" and x[1:].isdigit():
            return "%%%d" % (24 + int(x[1:]))
        if x[0] == "d" and x[1:].isdigit():
            return "%%%d" % (32 + int(x[1:]))
        return x

    for it in ins:
        lines.append("    %s %s;" % (it[0], ", ".join(opnd(x) for x in it[1:])))
    body = "\n".join('        "%s\\n\\t"' % ln.strip() for ln in ["{"] + lines + ["}"])
    outs = ", ".join('"=r"(r[%d])' % i for i in range(8))
    inps = ", ".join('"r"(a[%d])' % i for i in range(8))
    args = "uint32_t* r, const uint32_t* a"
    if n_in >= 2:
        inps += ", " + ", ".join('"r"(b[%d])' % i for i in range(8))
        args += ", const uint32_t* b"
    if n_in == 4:
        inps += ", " + ", ".join('"r"(c[%d])' % i for i in range(8)) + ", " + ", ".join('"r"(d[%d])' % i for i in range(8))
        args += ", const uint32_t* c, const uint32_t* d"
    return ("__device__ __forceinline__ void %s(%s) {\n    asm(\n%s\n        : %s\n        : %s);\n}\n"
            % (fname, args, body, outs, inps))


def main():
    out = ["// GENERATED by fp_gen.py -- do not edit.  Every instruction list below was executed by the generator's",
           "// PTX interpreter against Python bigints (edge + random operands) before this file was written.",
           "#pragma once", "#include <stdint.h>", "#if defined(__CUDA_ARCH__)", ""]
    for name, mod in FIELDS.items():
        n = check(name, mod)
        print("%s: verified; instruction counts mul/add/sub/mul2/sqr = %s" % (name, n))
        out.append(emit_fn("%s_mul_ptx" % name, gen_mul(mod), 2))
        out.append(emit_fn("%s_add_ptx" % name, gen_add(mod), 2))
        out.append(emit_fn("%s_sub_ptx" % name, gen_sub(mod), 2))
        out.append(emit_fn("%s_mul2_ptx" % name, gen_mul2(mod), 4))
        out.append(emit_fn("%s_sqr_ptx" % name, gen_sqr(mod), 1))
    out.append("#endif  // __CUDA_ARCH__")
    if "--check" not in sys.argv:
        import os
        with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "fp_ptx.cuh"), "w") as f:
            f.write("\n".join(out) + "\n")


if __name__ == "__main__":
    main()
