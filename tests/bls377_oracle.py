"""BLS12-377 for the CPU oracle (test infrastructure only): the curve parameters, Fq2 = Fq[u]/(u^2 + 5), the textbook
ate pairing over Fq12 = Fq[w]/(w^12 + 5), ark-ec's SWFlags wire form, Tonelli-Shanks square roots, and the cofactors and
small torsion of both groups.

`oracle/` states BLS12-381 and BN254; this module adds the third curve beside it without changing it.  Importing it
registers BLS12-377's groups with `oracle.ec.groups` and its pairing engine with `oracle.pairing.engine`, so the generic
oracle code (MSM, NTT, R1CS, Groth16 setup / prove / verify) runs on it unchanged.

Everything is derived from the seed x = 0x8508c00000000001 and checked in tests/test_oracle_bls12_377.py: r = x^4 - x^2 + 1,
p = (x - 1)^2 r / 3 + x, generators on their curves and of order r, the GT exponent of the kernels' pairing (k = 3).
"""
from oracle import ec as _ec
from oracle import pairing as _pairing
from oracle.params import Curve

X = 0x8508C00000000001
P = (X - 1) ** 2 * (X ** 4 - X ** 2 + 1) // 3 + X
R = X ** 4 - X ** 2 + 1
NR = -5                                  # u^2 = NR in Fq2
B2 = (0, (-pow(5, -1, P)) % P)           # 1 / u: G2 is the D-type twist y^2 = x^3 + 1 / u

BLS12_377 = Curve(
    name="bls12_377",
    curve_id=2,
    p=P,
    r=R,
    b=1,
    b2=B2,
    g1=(
        81937999373150964239938255573465948239988671502647976594219695644855304257327692006745978603320413799295628339695,
        241266749859715473739788878240585681733927191168601896383759122102112907357779751001206799952863815012735208165030,
    ),
    g2=(
        (
            233578398248691099356572568220835526895379068987715365179118596935057653620464273615301663571204657964920925606294,
            140913150380207355837477652521042157274541796891053068589147167627541651775299824604154852141315666357241556069118,
        ),
        (
            63160294768292073209381361943935198908131692476676907196754037919244929611450776219210369229519898517858833747423,
            149157405641012693445398062341192467754805999074082136895788947234480009303640899064710353187729182149407503257491,
        ),
    ),
    fr_generator=22,
    fr_two_adicity=47,
    fq_limbs64=6,
)

# #E(Fq) = h1 r and #E'(Fq2) = h2 r (BLS12 family polynomials in x)
H1 = (X - 1) ** 2 // 3
H2 = (X ** 8 - 4 * X ** 7 + 5 * X ** 6 - 4 * X ** 4 + 6 * X ** 3 - 4 * X ** 2 - 4 * X + 13) // 9


def two_adicity(n):
    k = 0
    while n % 2 == 0:
        n, k = n // 2, k + 1
    return k


def small_primes(n, bound=20000):
    """the primes below `bound` dividing n"""
    out = []
    for q in range(2, bound):
        if all(q % d for d in range(2, int(q ** 0.5) + 1)) and n % q == 0:
            out.append(q)
    return out


# ---- fields --------------------------------------------------------------------------------------------------------
class Fld5(_ec.Fld):
    """Fq2 = Fq[u]/(u^2 + 5) in the oracle's field interface"""

    def mul(self, a, b):
        p = self.p
        return ((a[0] * b[0] + NR * a[1] * b[1]) % p, (a[0] * b[1] + a[1] * b[0]) % p)

    def inv(self, a):
        p = self.p
        n = pow(a[0] * a[0] - NR * a[1] * a[1], -1, p)
        return (a[0] * n % p, (-a[1]) * n % p)


def sqrt_fq(a, p=P):
    """Tonelli-Shanks: a square root of a mod p, or None"""
    a %= p
    if a == 0:
        return 0
    if pow(a, (p - 1) // 2, p) != 1:
        return None
    s, q = two_adicity(p - 1), (p - 1) >> two_adicity(p - 1)
    z = next(g for g in range(2, p) if pow(g, (p - 1) // 2, p) == p - 1)
    m, c, t, x = s, pow(z, q, p), pow(a, q, p), pow(a, (q + 1) // 2, p)
    while t != 1:
        i, t2 = 0, t
        while t2 != 1:
            t2, i = t2 * t2 % p, i + 1
        b = pow(c, 1 << (m - i - 1), p)
        m, c, t, x = i, b * b % p, t * b * b % p, x * b % p
    return x


def sqrt_fq2(a, p=P):
    """a square root in Fq[u]/(u^2 + 5) by the norm method, or None"""
    F = Fld5(p, 2)
    a0, a1 = a[0] % p, a[1] % p
    if a1 == 0:
        s = sqrt_fq(a0, p)
        if s is not None:
            return (s, 0)
        s = sqrt_fq(-a0 * pow(5, -1, p), p)
        return None if s is None else (0, s)
    alpha = sqrt_fq(a0 * a0 + 5 * a1 * a1, p)
    if alpha is None:
        return None
    half = pow(2, -1, p)
    x0 = sqrt_fq((a0 + alpha) * half, p)
    if x0 is None:
        x0 = sqrt_fq((a0 - alpha) * half, p)
    if x0 is None:
        return None
    y = (x0, a1 * pow(2 * x0, -1, p) % p)
    return y if F.sqr(y) == (a0, a1) else None


def _register_groups():
    if BLS12_377.name not in _ec._cache:
        _ec._cache[BLS12_377.name] = (
            _ec.Group(_ec.Fld(P, 1), BLS12_377.b, BLS12_377.g1, R),
            _ec.Group(Fld5(P, 2), B2, BLS12_377.g2, R),
        )


_register_groups()


def groups():
    return _ec.groups(BLS12_377)


# ---- pairing -------------------------------------------------------------------------------------------------------
def _make_fq12(p, mod0):
    """Fq[w] / (w^12 - mod0) over coefficient lists (w^6 = u, u^2 = -5: mod0 = -5)"""

    class Fq12:
        __slots__ = ("c",)

        def __init__(self, coeffs):
            self.c = [x % p for x in coeffs] + [0] * (12 - len(coeffs))

        @staticmethod
        def one():
            return Fq12([1])

        @staticmethod
        def zero():
            return Fq12([0])

        def __eq__(self, o):
            return self.c == o.c

        def is_zero(self):
            return not any(self.c)

        def __add__(self, o):
            return Fq12([a + b for a, b in zip(self.c, o.c)])

        def __sub__(self, o):
            return Fq12([a - b for a, b in zip(self.c, o.c)])

        def __neg__(self):
            return Fq12([-a for a in self.c])

        def scale(self, k):
            return Fq12([a * k for a in self.c])

        def __mul__(self, o):
            t = [0] * 23
            for i, ai in enumerate(self.c):
                if ai:
                    for j, bj in enumerate(o.c):
                        t[i + j] += ai * bj
            for k in range(22, 11, -1):
                t[k - 12] += mod0 * t[k]
            return Fq12(t[:12])

        def sqr(self):
            return self * self

        def pow(self, e):
            out, base = Fq12.one(), self
            while e:
                if e & 1:
                    out = out * base
                base = base * base
                e >>= 1
            return out

        def inv(self):
            """extended Euclid on polynomials over Fq against w^12 - mod0"""
            def trim(a):
                while len(a) > 1 and a[-1] == 0:
                    a = a[:-1]
                return a

            def divmod_(a, b):
                a, q = list(a), [0] * max(1, len(a) - len(b) + 1)
                ib = pow(b[-1], -1, p)
                for i in range(len(a) - len(b), -1, -1):
                    f = a[i + len(b) - 1] * ib % p
                    q[i] = f
                    for j, bj in enumerate(b):
                        a[i + j] = (a[i + j] - f * bj) % p
                return trim(q), trim(a[: len(b) - 1] or [0])

            def mul(a, b):
                t = [0] * (len(a) + len(b) - 1)
                for i, x in enumerate(a):
                    for j, y in enumerate(b):
                        t[i + j] = (t[i + j] + x * y) % p
                return trim(t)

            def sub(a, b):
                n = max(len(a), len(b))
                return trim([((a[i] if i < len(a) else 0) - (b[i] if i < len(b) else 0)) % p for i in range(n)])

            r0, r1 = [(-mod0) % p] + [0] * 11 + [1], trim(list(self.c))
            s0, s1 = [0], [1]
            while r1 != [0]:
                q, rem = divmod_(r0, r1)
                r0, r1 = r1, rem
                s0, s1 = s1, sub(s0, mul(q, s1))
            assert len(r0) == 1, "not invertible"
            ic = pow(r0[0], -1, p)
            return Fq12([x * ic for x in s0[:12]])

        def __truediv__(self, o):
            return self * o.inv()

    return Fq12


class Engine377(_pairing.Engine):
    """The oracle's textbook ate pairing with BLS12-377's tower: w^6 = u, u^2 = -5, D-type twist, loop over x"""

    def __init__(self):
        self.curve = BLS12_377
        self.P, self.R = P, R
        self.xi0 = 0                         # w^6 = u
        self.loop = X                        # T = t - 1 = x
        self.Fq12 = _make_fq12(P, NR)
        w = self.Fq12([0, 1])
        self.tx, self.ty = w * w, w * w * w  # untwist (x w^2, y w^3)


def engine():
    if BLS12_377.name not in _pairing._ENGINES:
        _pairing._ENGINES[BLS12_377.name] = Engine377()
    return _pairing._ENGINES[BLS12_377.name]


engine()

K = 3   # e = oracle^K for the kernels' pairing (pairing.cuh): the same Miller function, hard part times 3, no conjugation
W_POWERS = [0, 2, 4, 1, 3, 5]   # coefficient of w^k at position k of ark's Fp12 layout


def gt_to_oracle(arr):
    """uint32 limbs of Fq12 elements (ark layout, Montgomery) -> oracle Fq12; a + bu at w^k is a w^k + b w^(k+6)"""
    from tests.util import unpack_u32

    rinv = pow(1 << 384, -1, P)
    vals = [v * rinv % P for v in unpack_u32(arr, 12)]
    E = engine()
    out = []
    for e in range(len(vals) // 12):
        v = vals[12 * e: 12 * e + 12]
        co = [0] * 12
        for slot, k in enumerate(W_POWERS):
            co[k], co[k + 6] = v[2 * slot], v[2 * slot + 1]
        out.append(E.Fq12(co))
    return out


def gt_from_oracle(elems):
    from tests.util import pack_u32

    flat = []
    for e in elems:
        for k in W_POWERS:
            flat += [e.c[k] * (1 << 384) % P, e.c[k + 6] * (1 << 384) % P]
    return pack_u32(flat, 12)


# ---- ark-ec SWFlags wire form (little-endian, G2 as c0 || c1, flags in the top byte of the last element) -------------
FQ_BYTES = 48


def _larger(y):
    """y > -y as canonical integers (Fq2: c1 first, then c0)"""
    if isinstance(y, tuple):
        n = ((-y[0]) % P, (-y[1]) % P)
        return (y[1], y[0]) > (n[1], n[0])
    return y > (-y) % P


def encode_point(group, Pt, compressed=True):
    coord = FQ_BYTES * group
    out = bytearray(coord * (1 if compressed else 2))
    if Pt is None:
        out[-1] |= 0x40
        return bytes(out)

    def put(off, v):
        vals = [v] if group == 1 else list(v)
        for i, c in enumerate(vals):
            out[off + i * FQ_BYTES: off + (i + 1) * FQ_BYTES] = c.to_bytes(FQ_BYTES, "little")

    put(0, Pt[0])
    if not compressed:
        put(coord, Pt[1])
    if _larger(Pt[1]):
        out[-1] |= 0x80
    return bytes(out)


def decode_point(group, data, compressed=True, validate=True):
    """-> (status, point) with status as deserialize.cuh's DecodeStatus: 0 ok, 1 flags, 2 non-canonical, 3 not on the
    curve, 4 not in the subgroup"""
    G = groups()[group - 1]
    coord = FQ_BYTES * group
    data = bytearray(data)
    flags = data[-1] & 0xC0
    data[-1] &= 0x3F
    if flags == 0xC0:
        return 1, None

    def get(off):
        vals = [int.from_bytes(data[off + i * FQ_BYTES: off + (i + 1) * FQ_BYTES], "little") for i in range(group)]
        return vals

    xs = get(0)
    ys = get(coord) if not compressed else [0] * group
    if flags & 0x40:
        return (0, None) if not any(xs) and not any(ys) else (1, None)
    if any(v >= P for v in xs):
        return 2, None
    x = xs[0] if group == 1 else tuple(xs)
    rhs = G.f.add(G.f.mul(G.f.sqr(x), x), G.b)
    if compressed:
        y = sqrt_fq(rhs) if group == 1 else sqrt_fq2(rhs)
        if y is None:
            return 3, None
        if _larger(y) != bool(flags & 0x80):
            y = G.f.neg(y)
    else:
        if any(v >= P for v in ys):
            return 2, None
        y = ys[0] if group == 1 else tuple(ys)
        if validate and G.f.sqr(y) != rhs:
            return 3, None
    Pt = (x, y)
    if validate and not in_subgroup(group, Pt):
        return 4, None
    return 0, Pt


def mul_unreduced(G, Pt, k):
    """k P without reducing k mod r (the oracle's Group.mul reduces it)"""
    acc = G.to_jac(None)
    J = G.to_jac(Pt)
    for bit in bin(k)[2:]:
        acc = G.jdbl(acc)
        if bit == "1":
            acc = G.jadd(acc, J)
    return G.to_affine(acc)


def in_subgroup(group, Pt):
    return Pt is None or mul_unreduced(groups()[group - 1], Pt, R) is None


def random_curve_point(group, rng):
    """a uniformly random point of E(Fq) / E'(Fq2), generally outside the subgroup"""
    G = groups()[group - 1]
    while True:
        x = rng.randrange(P) if group == 1 else (rng.randrange(P), rng.randrange(P))
        rhs = G.f.add(G.f.mul(G.f.sqr(x), x), G.b)
        y = sqrt_fq(rhs) if group == 1 else sqrt_fq2(rhs)
        if y is not None:
            return (x, y)


def torsion_point(group, q, rng):
    """a point of order exactly q for a prime q dividing the cofactor"""
    G = groups()[group - 1]
    h = H1 if group == 1 else H2
    qe = q
    while h % (qe * q) == 0:
        qe *= q
    while True:
        T = mul_unreduced(G, random_curve_point(group, rng), h * R // qe)   # in the q-power torsion
        if T is None:
            continue
        while mul_unreduced(G, T, q) is not None:
            T = mul_unreduced(G, T, q)
        return T
