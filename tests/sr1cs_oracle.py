"""A numpy restatement of Sr1csAdapter::r1cs_to_sr1cs_with_assignment (relations/src/sr1cs/mod.rs:191-265) on CSR arrays.

The reference walks the rows in order and gives each column other than ONE the next new witness the first time it meets
it (A_i, B_i, C_i in stored order), then the square s_i of the row.  Here every term gets its scan key -- its position in
the concatenation of every row's A, B, C terms and square slot -- and np.unique over the keys' columns finds each
column's first key; the witness numbers are the ranks of those keys among the allocation events.  Everything except field
products is vectorised, so it runs at 2^24 rows; coefficients stay Montgomery limbs (uint32 x 8), and the only big-int
work is per distinct coefficient value, per repeated (row, column) pair, and per square asked for."""
import numpy as np

R = 1 << 256


def limbs_to_ints(a, words=8):
    """(n * words) uint32 limbs -> list of Python ints"""
    b = np.ascontiguousarray(a, dtype=np.uint32).tobytes()
    n = 4 * words
    return [int.from_bytes(b[i:i + n], "little") for i in range(0, len(b), n)]


def ints_to_limbs(xs):
    return np.frombuffer(b"".join(v.to_bytes(32, "little") for v in xs), dtype=np.uint32).copy()


def map_values(r, limbs, f):
    """f applied to every coefficient (Montgomery ints mod r), computed once per distinct value"""
    v = np.ascontiguousarray(np.asarray(limbs, dtype=np.uint32).reshape(-1, 8))
    if v.shape[0] == 0:
        return np.zeros(0, dtype=np.uint32)
    u, inv = np.unique(v.view(np.dtype((np.void, 32))).ravel(), return_inverse=True)
    ui = limbs_to_ints(np.frombuffer(u.tobytes(), dtype=np.uint32))
    return ints_to_limbs([f(x) % r for x in ui]).reshape(-1, 8)[inv.ravel()].reshape(-1)


def canonical(r, n_rows, rows, col, coeff):
    """entries (row, col, Montgomery limbs) -> CSR sorted by column within each row, repeated columns summed, zero
    coefficients dropped: (row_ptr u64, col u32, coeff limbs u32)"""
    rows = np.asarray(rows, dtype=np.int64)
    col = np.asarray(col, dtype=np.int64)
    c = np.asarray(coeff, dtype=np.uint32).reshape(-1, 8)
    order = np.lexsort((col, rows))
    rows, col, c = rows[order], col[order], c[order]
    new = np.ones(rows.shape[0], dtype=bool)
    if rows.shape[0]:
        new[1:] = (rows[1:] != rows[:-1]) | (col[1:] != col[:-1])
    start = np.flatnonzero(new)
    size = np.diff(np.append(start, rows.shape[0]))
    out = c[start].copy()
    multi = np.flatnonzero(size > 1)
    if len(multi):
        # exact sums of the repeated groups in 64-bit limbs, carried into 9 words; mod r once per distinct sum
        s = np.zeros((len(start), 9), dtype=np.uint64)
        s[:, :8] = np.add.reduceat(c.astype(np.uint64), start, axis=0)
        s = s[multi]
        for i in range(8):
            s[:, i + 1] += s[:, i] >> np.uint64(32)
            s[:, i] &= np.uint64(0xFFFFFFFF)
        u, inv = np.unique(np.ascontiguousarray(s.astype(np.uint32)).view(np.dtype((np.void, 36))).ravel(), return_inverse=True)
        vals = ints_to_limbs([v % r for v in limbs_to_ints(np.frombuffer(u.tobytes(), dtype=np.uint32), 9)]).reshape(-1, 8)
        out[multi] = vals[inv.ravel()]
    keep = out.any(axis=1)
    rows, col, out = rows[start][keep], col[start][keep], out[keep]
    row_ptr = np.zeros(n_rows + 1, dtype=np.uint64)
    np.add.at(row_ptr, rows + 1, 1)
    return np.cumsum(row_ptr).astype(np.uint64), col.astype(np.uint32), out.reshape(-1)


def canonical_csr(r, row_ptr, col, coeff):
    n_rows = len(row_ptr) - 1
    rows = np.repeat(np.arange(n_rows, dtype=np.int64), np.diff(np.asarray(row_ptr, dtype=np.int64)))
    return canonical(r, n_rows, rows, col, coeff)


class Sr1cs:
    """The conversion of the R1CS csr = [(row_ptr, col, coeff limbs)] x 3 (A, B, C) with n_instance public columns (0 = ONE).
    Attributes: n_instance, n_witness, n_rows (of the result), pub (the used public columns p_k), ren (source column -> new
    column, 0 for ONE and unused ones), src_of (new column -> source column, -1 for a square), sq_col (row i -> column of
    s_i); matrices() gives the two arguments in canonical form."""

    def __init__(self, r, csr, n_instance):
        self.r, self.csr = r, csr
        rp = [np.asarray(m[0], dtype=np.int64) for m in csr]
        m = len(rp[0]) - 1
        self.m = m
        lens = [np.diff(x) for x in rp]
        base = rp[0][:-1] + rp[1][:-1] + rp[2][:-1] + np.arange(m, dtype=np.int64)
        before = [np.zeros(m, dtype=np.int64), lens[0], lens[0] + lens[1]]
        self.rows = [np.repeat(np.arange(m, dtype=np.int64), lens[k]) for k in range(3)]
        keys, cols = [], []
        for k in range(3):
            off = np.arange(len(self.rows[k]), dtype=np.int64) - rp[k][self.rows[k]]
            keys.append(base[self.rows[k]] + before[k][self.rows[k]] + off)
            cols.append(np.asarray(csr[k][1], dtype=np.int64))
        key, col = np.concatenate(keys), np.concatenate(cols)
        sq_key = base + lens[0] + lens[1] + lens[2]
        used = col != 0
        key, col = key[used], col[used]
        order = np.argsort(key, kind="stable")
        uniq, first_at = np.unique(col[order], return_index=True)   # first_at: the first (smallest-key) occurrence
        first_key = key[order][first_at]
        events = np.sort(np.concatenate([first_key, sq_key]))
        wnum = np.searchsorted(events, first_key)
        sq_w = np.searchsorted(events, sq_key)
        self.pub = uniq[uniq < n_instance]
        P = len(self.pub)
        self.n_instance, self.n_witness = 1 + P, len(uniq) + m
        self.n_rows = 2 * m + P
        n_src = int(max(col.max() + 1 if len(col) else 1, n_instance))
        self.ren = np.zeros(n_src, dtype=np.int64)
        self.ren[uniq] = 1 + P + wnum
        self.sq_col = 1 + P + sq_w
        n_vars = self.n_instance + self.n_witness
        self.src_of = np.full(n_vars, -1, dtype=np.int64)
        self.src_of[0] = 0
        self.src_of[1:1 + P] = self.pub
        self.src_of[1 + P + wnum] = uniq

    def matrices(self):
        """[(row_ptr, col, coeff limbs)] of L and R, canonical"""
        r, csr, m, P = self.r, self.csr, self.m, len(self.pub)
        one = ints_to_limbs([R % r])
        minus_one = ints_to_limbs([(r - R % r) % r])
        ren = lambda k: self.ren[np.asarray(csr[k][1], dtype=np.int64)]
        ra, rb, rc = self.rows
        a, b, c = (np.asarray(csr[k][2], dtype=np.uint32) for k in range(3))
        neg_b = map_values(r, b, lambda x: r - x)
        four_c = map_values(r, c, lambda x: 4 * x)
        k = np.arange(P, dtype=np.int64)
        L = canonical(r, self.n_rows,
                      np.concatenate([2 * ra, 2 * ra + 1, 2 * rb, 2 * rb + 1, 2 * m + k, 2 * m + k]),
                      np.concatenate([ren(0), ren(0), ren(1), ren(1), self.ren[self.pub], 1 + k]),
                      np.concatenate([a, a, b, neg_b, np.tile(one, P), np.tile(minus_one, P)]))
        i = np.arange(m, dtype=np.int64)
        Rm = canonical(r, self.n_rows,
                       np.concatenate([2 * rc, 2 * i, 2 * i + 1]),
                       np.concatenate([ren(2), self.sq_col, self.sq_col]),
                       np.concatenate([four_c, np.tile(one, 2 * m)]))
        return [L, Rm]

    def copied(self, z):
        """z' on every column that copies z (z: (n_assign, n_src * 8) limbs) -> (columns, their limbs); ONE is Montgomery 1"""
        z = np.asarray(z, dtype=np.uint32).reshape(z.shape[0], -1, 8)
        cols = np.flatnonzero(self.src_of >= 0)
        vals = z[:, self.src_of[cols], :].copy()
        vals[:, 0, :] = ints_to_limbs([R % self.r])
        return cols, vals

    def squares(self, z_row, rows):
        """s_i for the given rows of one assignment z_row (n_src * 8 limbs, Montgomery) -> Montgomery ints"""
        r, csr = self.r, self.csr
        zi = np.asarray(z_row, dtype=np.uint32).reshape(-1, 8)
        Rinv = pow(R, -1, r)
        out = []
        for i in rows:
            acc = 0
            for k, sign in ((0, 1), (1, -1)):
                rp, col, co = csr[k]
                lo, hi = int(rp[i]), int(rp[i + 1])
                cs = limbs_to_ints(np.asarray(co, dtype=np.uint32)[8 * lo:8 * hi])
                for j, cm in zip(range(lo, hi), cs):
                    c0 = int(col[j])
                    v = 1 if c0 == 0 else limbs_to_ints(zi[c0])[0] * Rinv % r
                    acc += sign * (cm * Rinv % r) * v
            acc %= r
            out.append(acc * acc % r * R % r)
        return out

    def assignment(self, z):
        """every element of z' for z (n_assign, n_src * 8) -> (n_assign, n_vars * 8) limbs"""
        n = z.shape[0]
        out = np.zeros((n, self.n_instance + self.n_witness, 8), dtype=np.uint32)
        cols, vals = self.copied(z)
        out[:, cols, :] = vals
        for a in range(n):
            out[a, self.sq_col, :] = ints_to_limbs(self.squares(z[a], range(self.m))).reshape(-1, 8)
        return out.reshape(n, -1)


def check(r, mats, z_mont_ints):
    """which rows of the SR1CS (L, R canonical or not) z fails: L(z)^2 != R(z); z as Montgomery ints"""
    Rinv = pow(R, -1, r)
    z = [v * Rinv % r for v in z_mont_ints]
    (lrp, lcol, lco), (rrp, rcol, rco) = mats
    lc, rc = [c * Rinv % r for c in limbs_to_ints(lco)], [c * Rinv % r for c in limbs_to_ints(rco)]
    bad = []
    for i in range(len(lrp) - 1):
        lv = sum(lc[e] * z[int(lcol[e])] for e in range(int(lrp[i]), int(lrp[i + 1]))) % r
        rv = sum(rc[e] * z[int(rcol[e])] for e in range(int(rrp[i]), int(rrp[i + 1]))) % r
        if lv * lv % r != rv:
            bad.append(i)
    return bad
