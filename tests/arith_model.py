"""Exact-integer models of the word-level arithmetic of hexl_b200/csrc/ntt_kernels.cuh (no GPU).

Every function below restates one device function with the same 32-bit partial products, in Python integers
reduced mod 2^64 where the device wraps.  tests/test_arith_model.py checks the range and congruence claims the
kernels rely on (quotient estimates low by at most two, lazy ranges, the FAST-mode growth bounds) on adversarial
and random operands, independently of the GPU parity tests, which can only sample."""

M64 = (1 << 64) - 1
M32 = (1 << 32) - 1


def split(x):
    return x & M32, (x >> 32) & M32


def mulhi(a, b):
    return (a * b) >> 64


def mulhi_approx(a, b):
    """ntt_kernels.cuh:mulhi_approx -- a1*b1 + hi32(a1*b0) + hi32(a0*b1)"""
    a0, a1 = split(a)
    b0, b1 = split(b)
    hs = ((a1 * b0) >> 32) + ((a0 * b1) >> 32)
    return (a1 * b1 + hs) & M64


def shoup(w, q):
    return (w << 64) // q


def mad_chain(x, w, Q, q):
    """low 64 bits of x*w + Q*(2^64 - q)"""
    return (x * w + Q * ((1 << 64) - q)) & M64


def mul_tw(x, w, wp, q, approx):
    Q = mulhi_approx(x, wp) if approx else mulhi(x, wp)
    return mad_chain(x, w, Q, q)


def mu_of(q):
    return (1 << 64) // q


def barrett_lazy(x, q):
    return (x - mulhi(x, mu_of(q)) * q) & M64


def barrett_lazy_bigq(x, q):
    """q >= 2^32: mu fits one word; Q = hi32(x1*mu + hi32(x0*mu))"""
    mu0 = mu_of(q) & M32
    x0, x1 = split(x)
    s = x1 * mu0
    h = (x0 * mu0) >> 32
    Q = ((s + h) >> 32) & M32
    return (x + Q * ((1 << 64) - q)) & M64


def barrett_lazy3_bigq(x, q):
    mu0 = mu_of(q) & M32
    _, x1 = split(x)
    Q = (x1 * mu0) >> 32
    return (x + Q * ((1 << 64) - q)) & M64


def csub_s(x, b):
    d = (x - b) & M64
    return x if d >> 63 else d


def csub(x, b):
    return x - b if x >= b else x


def prod_constants(q):
    """capi.h:dyadic_modulus -- shift = bits(q) - 2, mu = floor(2^(shift + 64) / q)"""
    shift = q.bit_length() - 2
    return (1 << (shift + 64)) // q, shift


def prod_lazy(x, y, q, approx):
    """ntt_kernels.cuh:prod_lazy"""
    pmu, shift = prod_constants(q)
    assert pmu < (1 << 64)
    x0, x1 = split(x)
    y0, y1 = split(y)
    t = x0 * y0
    uu = x0 * y1 + (t >> 32)
    vv = x1 * y0 + (uu & M32)
    hi = x1 * y1 + (uu >> 32) + (vv >> 32)
    lo = ((vv & M32) << 32) | (t & M32)
    assert uu <= M64 and vv <= M64 and hi <= M64 and (hi << 64) | lo == x * y
    c1 = ((lo >> shift) | (hi << (64 - shift))) & M64 if shift else lo
    assert c1 == (x * y) >> shift, "c1 must not lose high bits"
    Q = mulhi_approx(c1, pmu) if approx else mulhi(c1, pmu)
    return (lo + Q * ((1 << 64) - q)) & M64


# FAST-mode inverse bookkeeping (ntt_kernels.cuh:inv_slot_bound / inv_stage_cover), in units of q
K_FAST_PROD, K_FAST_BOUND = 4, 8


def inv_slot_bound(K, low):
    if low == 0:
        return K_FAST_BOUND << K
    h = max(b for b in range(K) if low & (1 << b))
    return K_FAST_PROD << (K - 1 - h)


def inv_stage_cover(s):
    return K_FAST_BOUND << s


def simulate_inverse_pass_bounds(K, nslots=16):
    """Bounds (units of q) of every register slot through K unreduced GS stages starting below 8q:
    X' = X + Y, Y' = (X + cq - Y) * w -> < 4q.  Returns (slot bounds, largest transient, cover ok)."""
    b = [K_FAST_BOUND] * nslots
    worst, ok = 0, True
    for s in range(K):
        cq = inv_stage_cover(s)
        nb = list(b)
        for e in range(nslots):
            if e & (1 << s):
                continue
            x, y = b[e], b[e | (1 << s)]
            ok &= y <= cq                    # cq must cover every Y of the stage
            worst = max(worst, x + y, x + cq)
            nb[e] = x + y
            nb[e | (1 << s)] = K_FAST_PROD
        b = nb
    return b, worst, ok


# ---- SMALL mode (q < 2^30): one 32-bit word per value (ntt_kernels.cuh:mul_tw32 / csub32)
def csub32(x, c):
    return min(x, (x - c) & M32)


def mul_tw32(x, w, q):
    wp = (w << 32) // q
    Q = (x * wp) >> 32
    return (x * w + Q * ((1 << 32) - q)) & M32


# ---- Montgomery reduction with R = 2^r (eltwise.cu:MontParams::redc): hi:lo < q*R -> T / R mod q
def redc(hi, lo, q, r):
    mask = (1 << r) - 1
    ninv = (-pow(q, -1, 1 << r)) % (1 << r)
    mm = ((lo & mask) * ninv) & mask
    mq = mm * q
    t_lo = (lo + (mq & M64)) & M64
    t_hi = (hi + (mq >> 64) + (1 if t_lo < lo else 0)) & M64
    s = ((t_hi << (64 - r)) | (t_lo >> r)) & M64
    return csub(s, q)


# ---- element-wise generalised Barrett product (eltwise.cu:FMult): inputs < in_mf*q
def reduce_from(x, q, k):
    if k >= 8:
        x = csub(x, q << 2)
    if k >= 4:
        x = csub(x, q << 1)
    if k >= 2:
        x = csub(x, q)
    return x


def eltwise_mult(a, b, q, in_mf):
    """z < 2q while bits(q) <= 61; at 62 bits (shift = 60) z < 3q and a second conditional subtraction follows"""
    x, y = reduce_from(a, q, in_mf), reduce_from(b, q, in_mf)
    pmu, shift = prod_constants(q)
    u = x * y
    lo, hi = u & M64, u >> 64
    c1 = ((lo >> shift) | (hi << (64 - shift))) & M64 if shift else lo
    z = csub((lo - mulhi(c1, pmu) * q) & M64, q)
    return csub(z, q) if shift == 60 else z


# ---- key-switch glue (seal.cu)
def shoup_lazy(x, w, q):
    return (x * w - mulhi(x, shoup(w, q)) * q) & M64


def ks_mac_digits_per_launch(q):
    """capi_keyswitch.cu:ks_mac_digits_per_launch -- digits one ks_mac_kernel launch adds up for moduli up to q: each product is
    a lazy transform output (< 4q) times a key word (< q), and their sum must stay below 2^128"""
    return min(64, ((1 << 128) - 1) // ((4 * q - 1) * (q - 1)))


def ks_mac_finish(acc, q):
    """ks_mac_kernel's tail: a 128-bit accumulator hi:lo -> [0, q):  hi * (2^64 mod q) + lo, both lazily"""
    hi, lo = acc >> 64, acc & M64
    v = (shoup_lazy(hi, (1 << 64) % q, q) + barrett_lazy(lo, q)) & M64
    assert v < 4 * q
    return csub(csub(v, q << 1), q)


def ks_finish(prod, t_ntt, modswitch, q):
    """ks_finish_kernel: (prod + 4q - t_ntt) * modswitch mod q for prod < q, t_ntt < 4q"""
    x = (prod + (q << 2) - t_ntt) & M64
    x = reduce_from(x, q, 8)
    return csub(shoup_lazy(x, modswitch, q), q)
