"""Executable specification of the register-resident DCT kernels (csrc/bk_fft_fast.cuh), written thread by thread.

Two real lines x1, x2 of length n = 2^LOGN form one complex line z = v1 + i v2 after Makhoul's reordering
(v[m] = x[2m], v[n-1-m] = x[2m+1]); one complex FFT of length n then yields both DCT-IIs:
    V1[k] = (Z[k] + conj Z[n-k]) / 2,  V2[k] = (Z[k] - conj Z[n-k]) / (2i),  C_p[k] = Re(w_k V_p[k]),  w_k = exp(-i pi k / 2n).
Every thread owns E elements; pass p of the DIF FFT has radix r_p <= E (a thread runs E / r_p butterflies in registers),
the array lives IN PLACE in shared memory between passes (butterfly (blk, b) of a pass with block length N_p = r M' touches
positions blk N_p + a M' + b, a < r), so Z[k] ends up at the digit-reversed position pos(k).
This file checks the index maps, the twiddle tables, the pair split and the fused (forward, divide by symbol, inverse)
middle step against scipy.fft, and counts shared-memory wavefronts for a padding function.

    python tools/fftcheck/model.py
"""
import numpy as np
import scipy.fft as sf


def radices(n, E):
    r = []
    rem = n
    while rem > 1:
        q = min(E, rem)
        r.append(q)
        rem //= q
    return r


def brev(j, r):
    b = r.bit_length() - 1
    return int(format(j, "0%db" % b)[::-1], 2) if b else 0


def bfly_fwd(a):
    """in-register radix-R DIF, in place; output q lands at index brev(q)"""
    R = len(a)
    if R == 1:
        return
    h = R // 2
    for i in range(h):
        t = a[i] - a[i + h]
        a[i] = a[i] + a[i + h]
        a[i + h] = t * np.exp(-2j * np.pi * i / R)
    lo, hi = a[:h].copy(), a[h:].copy()
    bfly_fwd(lo)
    bfly_fwd(hi)
    a[:h], a[h:] = lo, hi


def bfly_inv(a):
    """mirror: input Y_q at index brev(q), output natural, unnormalised inverse DFT"""
    R = len(a)
    if R == 1:
        return
    h = R // 2
    lo, hi = a[:h].copy(), a[h:].copy()
    bfly_inv(lo)
    bfly_inv(hi)
    a[:h], a[h:] = lo, hi
    for i in range(h):
        t = a[i + h] * np.exp(2j * np.pi * i / R)
        a[i + h] = a[i] - t
        a[i] = a[i] + t


class Plan:
    def __init__(self, n, E):
        self.n, self.E = n, E
        self.rad = radices(n, E)
        self.T = n // E
        # per-pass geometry
        self.Np, self.Mp = [], []
        N = n
        for r in self.rad:
            self.Np.append(N)
            self.Mp.append(N // r)
            N //= r
        # pos <-> k
        self.k_of_pos = np.zeros(n, dtype=int)
        for p in range(n):
            rem, k, w = p, 0, 1
            for r, M in zip(self.rad, self.Mp):
                q = rem // M
                rem -= q * M
                k += q * w
                w *= r
            self.k_of_pos[p] = k
        self.pos_of_k = np.argsort(self.k_of_pos)
        # per-pass contiguous twiddle tables: tw[p][(q-1) * M' + b] = W_{N_p}^{b q}
        self.tw = []
        for r, N, M in zip(self.rad, self.Np, self.Mp):
            t = np.zeros((r - 1) * M, dtype=complex)
            for q in range(1, r):
                for b in range(M):
                    t[(q - 1) * M + b] = np.exp(-2j * np.pi * b * q / N)
            self.tw.append(t)
        self.omega_pos = np.exp(-1j * np.pi * self.k_of_pos / (2 * n))  # w_k in position order

    def positions(self, p, tau, u):
        """positions touched by butterfly u of thread tau in pass p, in register order j (output q = brev(j))"""
        r, N, M = self.rad[p], self.Np[p], self.Mp[p]
        beta = tau + self.T * u
        blk, b = divmod(beta, M)
        return [blk * N + a * M + b for a in range(r)], b

    def forward(self, z):
        """z natural order (length n) -> smem array A with Z[k] at pos(k); returns (A, per-thread registers of the last pass)"""
        n, E, T = self.n, self.E, self.T
        A = z.astype(complex).copy()
        regs = np.zeros((T, E), dtype=complex)
        for p, r in enumerate(self.rad):
            out = A.copy()
            for tau in range(T):
                for u in range(E // r):
                    pos, b = self.positions(p, tau, u)
                    a = A[pos].copy()  # register j holds input a = j
                    bfly_fwd(a)
                    for j in range(r):
                        q = brev(j, r)
                        if q > 0 and self.Mp[p] > 1:
                            a[j] *= self.tw[p][(q - 1) * self.Mp[p] + b]
                        out[pos[q]] = a[j]
                        regs[tau, u * r + j] = a[j]
            A = out
        return A, regs

    def inverse(self, A):
        """A holds Zhat[k] at pos(k) -> natural order n * ifft"""
        for p in reversed(range(len(self.rad))):
            r = self.rad[p]
            out = A.copy()
            for tau in range(self.T):
                for u in range(self.E // r):
                    pos, b = self.positions(p, tau, u)
                    a = np.zeros(r, dtype=complex)
                    for j in range(r):
                        q = brev(j, r)
                        v = A[pos[q]]
                        if q > 0 and self.Mp[p] > 1:
                            v = v * np.conj(self.tw[p][(q - 1) * self.Mp[p] + b])
                        a[j] = v
                    bfly_inv(a)
                    for i in range(r):
                        out[pos[i]] = a[i]
            A = out
        return A


def makhoul(x):
    n = len(x)
    v = np.zeros(n, dtype=x.dtype)
    v[: n // 2] = x[0::2]
    v[n // 2:] = x[1::2][::-1]
    return v


def unmakhoul(v):
    n = len(v)
    x = np.zeros(n, dtype=v.dtype)
    x[0::2] = v[: n // 2]
    x[1::2] = v[n // 2:][::-1]
    return x


def dct_pair_forward(pl, x1, x2):
    """returns 2*C1, 2*C2 (the kernels leave out the 1/2 of the pair split) in natural k order"""
    n = pl.n
    z = makhoul(x1) + 1j * makhoul(x2)
    A, _ = pl.forward(z)
    C1, C2 = np.zeros(n), np.zeros(n)
    for p in range(n):
        k = pl.k_of_pos[p]
        Zk, Zc = A[p], np.conj(A[pl.pos_of_k[(n - k) % n]])
        V1, V2 = Zk + Zc, -1j * (Zk - Zc)
        w = pl.omega_pos[p]
        C1[k] = (w * V1).real
        C2[k] = (w * V2).real
    return C1, C2


def dct_pair_inverse(pl, C1, C2):
    """inverse of the unnormalised DCT-II (x n): x = C0 + 2 sum C_k cos"""
    n = pl.n
    A = np.zeros(n, dtype=complex)
    for p in range(n):
        k = pl.k_of_pos[p]
        c1n = C1[n - k] if k > 0 else 0.0
        c2n = C2[n - k] if k > 0 else 0.0
        # conj(w) (C1[k] - i C1[n-k]) + i conj(w) (C2[k] - i C2[n-k]) = conj(w) ((C1[k] + C2[n-k]) + i (C2[k] - C1[n-k]))
        A[p] = np.conj(pl.omega_pos[p]) * ((C1[k] + c2n) + 1j * (C2[k] - c1n))
    v = pl.inverse(A)
    return unmakhoul(v.real), unmakhoul(v.imag)


def fused_pair(pl, x1, x2, s1, s2):
    """forward, multiply C_p[k] by s_p[k] (s includes every normalisation), inverse -- the pair split done per position with the
    partner Z[n-k] read from shared memory, exactly as the kernel does"""
    n = pl.n
    z = makhoul(x1) + 1j * makhoul(x2)
    A, _ = pl.forward(z)
    B = np.zeros(n, dtype=complex)
    for p in range(n):
        k = pl.k_of_pos[p]
        nk = (n - k) % n
        Zk, Zc = A[p], np.conj(A[pl.pos_of_k[nk]])
        w = pl.omega_pos[p]
        A1, A2 = w * (Zk + Zc), w * (-1j) * (Zk - Zc)  # 2 (C_p[k] - i C_p[n-k])
        h1 = A1.real * s1[k] + 1j * A1.imag * s1[nk]    # s[n] never matters: Im A(0) = 0
        h2 = A2.real * s2[k] + 1j * A2.imag * s2[nk]
        B[p] = np.conj(w) * (h1 + 1j * h2)
    v = pl.inverse(B)
    return unmakhoul(v.real), unmakhoul(v.imag)


# ---- periodic transforms (BK_SH2D_PERIODIC): k_contig MODE 2 / 3 and k_strided MODE 3 -------------------------------------
def rfft_pair(pl, x1, x2):
    """k_contig MODE 2: two real rows form z = x1 + i x2 (natural order, no Makhoul reordering); per position the partner read
    splits Z into X1 = (Z[k] + conj Z[n-k]) / 2, X2 = (Z[k] - conj Z[n-k]) / 2i, stored as packed half-spectra
    [Re X0, Re X_{n/2}, Re X1, Im X1, ..., Re X_{n/2-1}, Im X_{n/2-1}]."""
    n = pl.n
    A, _ = pl.forward(x1 + 1j * x2)
    P1, P2 = np.zeros(n), np.zeros(n)
    for p in range(n):
        k = pl.k_of_pos[p]
        Zk, Zc = A[p], np.conj(A[pl.pos_of_k[(n - k) % n]])
        X1, X2 = (Zk + Zc) / 2, (Zk - Zc) / 2j
        if k == 0:
            P1[0], P2[0] = X1.real, X2.real
        elif k == n // 2:
            P1[1], P2[1] = X1.real, X2.real
        elif k < n // 2:
            P1[2 * k], P1[2 * k + 1] = X1.real, X1.imag
            P2[2 * k], P2[2 * k + 1] = X2.real, X2.imag
    return P1, P2


def unpack(P, k):
    """X[k] of a packed half-spectrum, any 0 <= k < n (X[n-k] = conj X[k])"""
    n = len(P)
    kk = k if k <= n // 2 else n - k
    if kk == 0 or kk == n // 2:
        return complex(P[1 if kk else 0], 0.0)
    x = complex(P[2 * kk], P[2 * kk + 1])
    return x if k == kk else np.conj(x)


def irfft_pair(pl, P1, P2):
    """k_contig MODE 3 before its epilogue: Z[k] = X1[k] + i X2[k] at every position, inverse passes -> n x1, n x2"""
    n = pl.n
    A = np.zeros(n, dtype=complex)
    for p in range(n):
        k = pl.k_of_pos[p]
        A[p] = unpack(P1, k) + 1j * unpack(P2, k)
    v = pl.inverse(A)
    return v.real, v.imag


def periodic_y_pair(pl, c0, c1, s0, sn=None):
    """k_strided MODE 3 on one column pair of length n (s includes every normalisation).  sn is None: the pair is the complex
    line c0 + i c1 of one kx, multiplied by s0[k].  Otherwise the pair holds the two real lines kx = 0 (symbol s0) and
    kx = Nx/2 (symbol sn): Z'[k] = ((s0 + sn)/2) Z[k] + ((s0 - sn)/2) conj Z[-k] with the partner read.  Returns n x."""
    n = pl.n
    A, _ = pl.forward(c0 + 1j * c1)
    B = np.zeros(n, dtype=complex)
    for p in range(n):
        k = pl.k_of_pos[p]
        if sn is None:
            B[p] = s0[k] * A[p]
        else:
            Zc = np.conj(A[pl.pos_of_k[(n - k) % n]])
            B[p] = 0.5 * (s0[k] + sn[k]) * A[p] + 0.5 * (s0[k] - sn[k]) * Zc
    v = pl.inverse(B)
    return v.real, v.imag


def periodic_apply(u, sym, E):
    """The whole BK_SH2D_PERIODIC pipeline on a (Ny, Nx) array: x r2c per row pair, y pass per column pair, x c2r per row pair.
    sym (Ny, Nx // 2 + 1) is the symbol over (ky, kx >= 0); the result is irfft2(rfft2(u) * sym)."""
    Ny, Nx = u.shape
    px, py = Plan(Nx, E), Plan(Ny, E)
    P = np.zeros((Ny, Nx))
    for j in range(0, Ny, 2):
        P[j], P[j + 1] = rfft_pair(px, u[j], u[j + 1])
    Q = np.zeros_like(P)
    scale = 1.0 / (Nx * Ny)
    for q in range(Nx // 2):
        if q == 0:
            a, b = periodic_y_pair(py, P[:, 0], P[:, 1], sym[:, 0] * scale, sym[:, Nx // 2] * scale)
        else:
            a, b = periodic_y_pair(py, P[:, 2 * q], P[:, 2 * q + 1], sym[:, q] * scale)
        Q[:, 2 * q], Q[:, 2 * q + 1] = a, b
    out = np.zeros_like(u)
    for j in range(0, Ny, 2):
        out[j], out[j + 1] = irfft_pair(px, Q[j], Q[j + 1])
    return out


def wavefronts(slots):
    """128-bit accesses are served per quarter warp (8 lanes x 16 B = 128 B): wavefronts = max lanes on one 16-byte bank group"""
    tot = 0
    for q in range(0, len(slots), 8):
        g = [s % 8 for s in slots[q:q + 8]]
        tot += max(np.bincount(g, minlength=8))
    return tot


def bank_report(pl, pad, pairs_interleaved=1):
    """average wavefronts per ideal wavefront for the in-place exchanges of every pass (lanes = consecutive tau of one pair,
    or interleaved with `pairs_interleaved` pairs whose arrays are n_pad apart)"""
    n, E, T = pl.n, pl.E, pl.T
    npad = pad(n - 1) + 1
    res = []
    for p, r in enumerate(pl.rad):
        tot = ideal = 0
        lanes = [(tau, pr) for tau in range(T) for pr in range(pairs_interleaved)]
        for w0 in range(0, len(lanes), 32):
            warp = lanes[w0:w0 + 32]
            for u in range(E // r):
                for a in range(r):
                    sl = []
                    for tau, pr in warp:
                        pos, _ = pl.positions(p, tau, u)
                        sl.append(pad(pos[a]) + pr * npad)
                    tot += wavefronts(sl)
                    ideal += (len(sl) + 7) // 8
        res.append(tot / ideal)
    return res


def bank_report_em(pl, pad, PP, nthreads=None):
    """Wavefronts per ideal wavefront of every pass (and of the partner read, last entry) for the layout the kernels use:
    thread tid = tau * PP + pr, slot(pos, pr) = pad(pos) * PP + pr  (element-major, pairs interleaved)."""
    n, E, T = pl.n, pl.E, pl.T
    nthreads = nthreads or min(T * PP, 256)
    lanes = [(tid // PP, tid % PP) for tid in range(nthreads)]
    slot = lambda pr, i: pad(i) * PP + pr
    res = []
    for p, r in enumerate(pl.rad):
        tot = ideal = 0
        for w0 in range(0, len(lanes), 32):
            warp = lanes[w0:w0 + 32]
            for u in range(E // r):
                for a in range(r):
                    sl = [slot(pr, pl.positions(p, tau, u)[0][a]) for tau, pr in warp]
                    tot += wavefronts(sl)
                    ideal += (len(sl) + 7) // 8
        res.append(tot / ideal)
    tot = ideal = 0
    rl = pl.rad[-1]
    for w0 in range(0, len(lanes), 32):
        warp = lanes[w0:w0 + 32]
        for u in range(E // rl):
            for j in range(rl):
                sl = []
                for tau, pr in warp:
                    pp = pl.positions(len(pl.rad) - 1, tau, u)[0][brev(j, rl)]
                    k = pl.k_of_pos[pp]
                    sl.append(slot(pr, pl.pos_of_k[(n - k) % n]))
                tot += wavefronts(sl)
                ideal += (len(sl) + 7) // 8
    res.append(tot / ideal)
    return res


def bank_report_natural(pl, padn, PP, nthreads=None):
    """Contiguous kernels: (scatter of the registers into the natural-order array nat[padn(k) * PP + pr], read k = tau + T i):
    wavefronts per ideal wavefront of both accesses."""
    n, E, T = pl.n, pl.E, pl.T
    nthreads = nthreads or min(T * PP, 256)
    lanes = [(tid // PP, tid % PP) for tid in range(nthreads)]
    rl, P = pl.rad[-1], len(pl.rad) - 1
    tot = ideal = 0
    for w0 in range(0, len(lanes), 32):
        warp = lanes[w0:w0 + 32]
        for u in range(E // rl):
            for j in range(rl):
                sl = [padn(pl.k_of_pos[pl.positions(P, tau, u)[0][brev(j, rl)]]) * PP + pr for tau, pr in warp]
                tot += wavefronts(sl)
                ideal += (len(sl) + 7) // 8
    w = tot / ideal
    tot = ideal = 0
    for w0 in range(0, len(lanes), 32):
        warp = lanes[w0:w0 + 32]
        for i in range(E):
            sl = [padn(i * T + tau) * PP + pr for tau, pr in warp]
            tot += wavefronts(sl)
            ideal += (len(sl) + 7) // 8
    return w, tot / ideal


if __name__ == "__main__":
    rng = np.random.default_rng(0)
    for n in (64, 128, 256, 512, 1024, 2048):
        for E in (8, 16, 32):
            if E > n:
                continue
            pl = Plan(n, E)
            x1, x2 = rng.standard_normal(n), rng.standard_normal(n)
            C1, C2 = dct_pair_forward(pl, x1, x2)
            r1 = sf.dct(x1, type=2)  # scipy: 2 sum x cos = 2 C
            r2 = sf.dct(x2, type=2)
            ef = max(np.abs(C1 - r1).max(), np.abs(C2 - r2).max()) / np.abs(r1).max()
            y1, y2 = dct_pair_inverse(pl, r1 / 2, r2 / 2)
            ei = max(np.abs(y1 / n - x1).max(), np.abs(y2 / n - x2).max())
            s1, s2 = rng.uniform(0.5, 2.0, n), rng.uniform(0.5, 2.0, n)
            f1, f2 = fused_pair(pl, x1, x2, s1 / (2 * n), s2 / (2 * n))
            g1 = sf.idct(sf.dct(x1, type=2) * s1, type=2)
            g2 = sf.idct(sf.dct(x2, type=2) * s2, type=2)
            eu = max(np.abs(f1 - g1).max(), np.abs(f2 - g2).max())
            pad = lambda i: i + (i >> 3)
            print(f"n={n:5d} E={E:2d} radices={pl.rad}  fwd {ef:.1e}  inv {ei:.1e}  fused {eu:.1e}   "
                  f"wavefront ratio pad i+i/8: {['%.2f' % v for v in bank_report(pl, pad)]}  none: {['%.2f' % v for v in bank_report(pl, lambda i: i)]}")
