"""CPU tier: a Python-integer model of ronk_ntt_any_u64's Bluestein path (ronkathon_b200/csrc/ntt_any.cu) — the chirp
exponents C(t, 2) mod n, the reflected spectrum r_s = v_((-s) mod N), the stepped runs of the chirp kernels (thread i of
a block takes t = base + i + 256·r) and the inverse's reversal — with the N-point cyclic convolution taken directly,
without a transform.  So it runs for every test prime, also those whose two-adicity rules the device path out
(p = 101, 17, 127), and is compared with the oracle's literal dft."""
import pytest

import oracle
from gpu_util import GL, MONT_PRIMES

THREADS, RUN = 256, 32     # AN_THREADS, AN_RUN
PRIMES = {**{k: (p, g) for k, (p, g, _) in MONT_PRIMES.items()}, "goldilocks": (GL, 7), "f101": (101, 2), "f17": (17, 14),
          "f127": (127, 3)}


def divisors(m, cap):
    return [d for d in range(1, cap + 1) if m % d == 0]


def conv_size(n):
    return 1 << (2 * n - 1 - 1).bit_length() if n > 1 else 1


def chirp_runs(p, w, n, length, scale=1):
    """scale · w^C(t,2) for t < length, produced as the kernels produce them: per thread a start by two powers, then
    z ← z·e, e ← e·w^(S²) along t, t + S, …; checked against the direct power at every t."""
    out = [None] * length
    S = THREADS
    step = pow(w, (S * S) % n, p)
    for base in range(0, length, S * RUN):
        for i in range(S):
            t = base + i
            if t >= length:
                break
            z = scale * pow(w, (t * (t - 1) // 2) % n, p) % p
            e = pow(w, (S * t + S * (S - 1) // 2) % n, p)
            for _ in range(RUN):
                if t >= length:
                    break
                out[t] = z
                z, e = z * e % p, e * step % p
                t += S
    for t in range(length):
        assert out[t] == scale * pow(w, (t * (t - 1) // 2) % n, p) % p, t
    return out


def bluestein(p, g, a, inverse=False):
    n = len(a)
    N = conv_size(n)
    w = pow(g, (p - 1) // n, p)
    winv = pow(w, p - 2, p)
    r = [0] * N                                          # anyntt_chirp_table: reflected, zero gap
    for t, v in enumerate(chirp_runs(p, w, n, 2 * n - 1)):
        r[(N - t) % N] = v
    cin = chirp_runs(p, winv, n, n)                      # anyntt_chirp_in: u_j, then zeros
    u = [int(a[j]) * cin[j] % p for j in range(n)] + [0] * (N - n)
    c = [sum(u[j] * r[(m - j) % N] for j in range(n)) % p for m in range(N)]   # the cyclic convolution
    scale = pow(n, p - 2, p) if inverse else 1           # anyntt_chirp_out
    cout = chirp_runs(p, winv, n, n, scale)
    out = [0] * n
    for t in range(n):
        out[(n - t) % n if inverse else t] = cout[t] * c[(N - t) % N] % p
    return out


@pytest.mark.parametrize("name", list(PRIMES))
def test_model_matches_dft(name):
    p, g = PRIMES[name]
    ns = divisors(p - 1, 300)
    ns = [n for n in ns if n & (n - 1)] or ns            # the power-of-two sizes take the transform itself
    for n in ns[:8] + ns[-4:]:
        a = oracle.splitmix(p, 100 + n, n)
        assert bluestein(p, g, a) == [int(v) for v in oracle.dft(p, a, g=g)], (name, n)
        ginv = pow(g, p - 2, p)
        ninv = pow(n, p - 2, p)
        exp = [int(v) * ninv % p for v in oracle.dft(p, a, g=ginv)]
        assert bluestein(p, g, a, inverse=True) == exp, (name, n)


def test_model_wraparound_and_runs():
    """The largest n for one N (2n - 1 = N - 1) and the smallest (2n - 1 just above N/2), with runs that cross the
    2n - 1 and n ends mid-block; the convolution's wrap must stay off the n words read."""
    p, g = GL, 7
    for n in (85, 255, 257):
        if (p - 1) % n:
            continue
        a = oracle.splitmix(p, n, n)
        got = bluestein(p, g, a)
        assert got == [int(v) for v in oracle.dft(p, a, g=g)], n
        assert [v * n % p for v in bluestein(p, g, got, inverse=True)] == [int(v) * n % p for v in a], n
