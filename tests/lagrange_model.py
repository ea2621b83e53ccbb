"""Python-integer model of the Lagrange-basis evaluation and opening on a coset s·H_n (ronk_poly_lagrange_eval_u64,
ronk_poly_lagrange_open_u64).  Nodes x_j = s·ω^j, ω = g^((p-1)/n); Z(X) = X^n - s^n; weights w_j = x_j / (n·s^n).
Importable without a GPU."""


def nodes(p, g, n, s=1):
    w = pow(g, (p - 1) // n, p)
    out, x = [], s % p
    for _ in range(n):
        out.append(x)
        x = x * w % p
    return out


def closed_form(p, g, y, x, s=1):
    """L(x) = Z(x) · Σ_j w_j y_j / (x - x_j); 0 at a node (the reference's l(x)·fold)."""
    n = len(y)
    sn = pow(s, n, p)
    zx = (pow(x, n, p) - sn) % p
    if zx == 0:
        return 0
    acc = 0
    for yj, xj in zip(y, nodes(p, g, n, s)):
        acc = (acc + int(yj) * xj * pow((x - xj) % p, -1, p)) % p
    return zx * pow(n * sn % p, -1, p) * acc % p


def value(p, g, y, z, s=1):
    """f(z): y_k at a node z = x_k, else the closed form."""
    xs = nodes(p, g, len(y), s)
    return int(y[xs.index(z)]) if z in xs else closed_form(p, g, y, z, s)


def quotient(p, g, y, z, s=1):
    """Evaluations on the nodes of (f - f(z)) / (X - z): (y_j - v) / (x_j - z), and at a node z = x_k,
    q_k = -x_k^-1 Σ_{j≠k} x_j q_j."""
    xs = nodes(p, g, len(y), s)
    v = value(p, g, y, z, s)
    q = [0 if xj == z else (int(yj) - v) * pow((xj - z) % p, -1, p) % p for yj, xj in zip(y, xs)]
    if z in xs:
        k = xs.index(z)
        q[k] = -pow(z, -1, p) * sum(xj * qj for xj, qj in zip(xs, q)) % p
    return v, q


def coefficients(p, g, y, s=1):
    """Monomial coefficients of the f with f(x_j) = y_j: a_i = s^-i / n · Σ_j y_j ω^(-ij).  O(n²)."""
    n = len(y)
    winv = pow(pow(g, (p - 1) // n, p), -1, p)
    ninv, sinv = pow(n, -1, p), pow(s, -1, p)
    out = []
    for i in range(n):
        acc, wi, t = 0, pow(winv, i, p), 1
        for yj in y:
            acc = (acc + int(yj) * t) % p
            t = t * wi % p
        out.append(acc * ninv * pow(sinv, i, p) % p)
    return out


def horner(p, c, x):
    acc = 0
    for v in reversed([int(u) for u in c]):
        acc = (acc * x + v) % p
    return acc
