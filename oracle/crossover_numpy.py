"""numpy mirror of the crossover post-pass (dsp_lp_crossover, dispatches_b200/csrc/dsp_crossover.cuh, DESIGN.md 4.6).

An independent implementation of the same rules on one LP  min c'x, A x = b, 0 <= x <= u  (A dense or scipy, u = inf where a column
has no bound): the same crash order, push, bounded primal / dual simplex with Harris' ratio test and the same tie-breaks, and the
artificials pivoted out by a dual ratio test.  The linear algebra is different on purpose: every solve with the basis matrix is an
LU solve of B (numpy.linalg.solve) from scratch, with no product-form inverse and no iterative refinement, so the mirror shares no
arithmetic with the kernel.  Returns dict(x, y, col_status [n] int8, row_basic [m] int8, status, pivots).
"""
from __future__ import annotations

import numpy as np

FEAS, PIVOT, BLAND_AFTER = 1e-9, 1e-7, 50
AT_LO, BASIC, AT_UP, INSIDE = 0, 1, 2, 3
OPTIMAL, MAX_ITER, NUMERICAL = 0, 1, 2


def crossover(A, b, c, u, x, max_pivots=0):
    A = np.asarray(A.toarray() if hasattr(A, "toarray") else A, float)
    m, n = A.shape
    b, c = np.asarray(b, float), np.asarray(c, float)
    u = np.maximum(np.asarray(u, float), 0.0)
    fin = np.isfinite(u)
    sp = max(1.0, np.abs(b).max(initial=0.0), np.abs(u[fin]).max(initial=0.0))
    sd = np.abs(c).max(initial=0.0) or 1.0
    tolp, told = FEAS * sp, FEAS * sd
    maxp = max_pivots if max_pivots > 0 else 10 * (m + n)
    Ae = np.hstack([A, np.eye(m)])                      # the artificials: unit columns with bounds [0, 0]
    ce = np.concatenate([c, np.zeros(m)])
    ue = np.concatenate([u, np.zeros(m)])
    stat = np.full(n + m, AT_LO)
    xv = np.zeros(n + m)
    x = np.asarray(x, float)
    for j in range(n):
        if x[j] <= tolp or u[j] <= 0.0:
            stat[j], xv[j] = AT_LO, 0.0
        elif u[j] - x[j] <= tolp:
            stat[j], xv[j] = AT_UP, u[j]
        else:
            stat[j], xv[j] = INSIDE, x[j]
    head = list(range(n, n + m))
    stat[n:] = BASIC
    B = lambda: Ae[:, head]
    # 1. crash: the inside columns, most interior first (ties by index)
    inside = [j for j in range(n) if stat[j] == INSIDE]
    inside.sort(key=lambda j: (-min(xv[j], u[j] - xv[j]), j))
    for j in inside:
        if all(h < n for h in head):
            break
        al = np.linalg.solve(B(), A[:, j])
        cand = [k for k in range(m) if head[k] >= n]
        k = min(cand, key=lambda k: (-abs(al[k]), k))
        if abs(al[k]) >= PIVOT * np.abs(A[:, j]).max():
            stat[head[k]] = AT_LO
            head[k] = j
            stat[j] = BASIC

    def solve_x():
        N = [j for j in range(n + m) if stat[j] != BASIC]
        xb = np.linalg.solve(B(), b - Ae[:, N] @ xv[N])
        xv[head] = xb

    def solve_y():
        y = np.linalg.solve(B().T, ce[head])
        return y, ce - Ae.T @ y

    def upper(v):
        return ue[v]

    def primal_ratio(al, direction, tol, bland):
        piv = PIVOT * np.abs(al).max()
        best = None
        for k in range(m):
            s = direction * al[k]
            if abs(s) < piv or s == 0.0:
                continue
            v = head[k]
            if s > 0:
                r = max(0.0, xv[v] + tol) / s
            elif np.isfinite(upper(v)):
                r = max(0.0, upper(v) - xv[v] + tol) / -s
            else:
                continue
            best = r if best is None else min(best, r)
        if best is None:
            return None
        cands = []
        for k in range(m):
            s = direction * al[k]
            if abs(s) < piv or s == 0.0:
                continue
            v = head[k]
            if s > 0:
                r = max(0.0, xv[v]) / s
            elif np.isfinite(upper(v)):
                r = max(0.0, upper(v) - xv[v]) / -s
            else:
                continue
            if r <= best:
                cands.append((0.0 if bland else -abs(s), v, k, r, s < 0))
        _, v, k, r, to_up = min(cands)
        return k, r, to_up

    def row_alpha(k):
        rho = np.linalg.solve(B().T, np.eye(m)[k])
        out = np.zeros(n)
        rmax = np.abs(rho).max()
        for j in range(n):
            if stat[j] == BASIC or u[j] <= 0.0:
                continue
            a = rho @ A[:, j]
            out[j] = a if abs(a) >= PIVOT * rmax * np.abs(A[:, j]).max() else 0.0
        return out

    def dual_ratio(alr, d, direction, bland):
        def ok(j):
            a = alr[j]
            if a == 0.0:
                return False
            lo = stat[j] == AT_LO
            return (lo and a * direction > 0) or (not lo and a * direction < 0)
        slack = lambda j: max(d[j], 0.0) if stat[j] == AT_LO else max(-d[j], 0.0)
        js = [j for j in range(n) if ok(j)]
        if not js:
            return None, None
        tmax = min((slack(j) + told) / abs(alr[j]) for j in js)
        q = min((j for j in js if slack(j) / abs(alr[j]) <= tmax), key=lambda j: (0.0 if bland else -abs(alr[j]), j))
        return q, slack(q) / abs(alr[q])

    def pivot(k, q, st, at):
        v = head[k]
        stat[v], xv[v] = st, at
        head[k] = q
        stat[q] = BASIC

    def dual_inf(j, d):
        if stat[j] == BASIC or u[j] <= 0.0:
            return 0.0
        if stat[j] == AT_LO and d[j] < -told:
            return -d[j]
        if stat[j] == AT_UP and d[j] > told:
            return d[j]
        return 0.0

    def primal_worst():
        best = None
        for k in range(m):
            v = head[k]
            viol = -xv[v] if xv[v] < -tolp else xv[v] - upper(v) if xv[v] > upper(v) + tolp else 0.0
            if viol > 0 and (best is None or (-viol, v) < (-best[0], best[1])):
                best = (viol, v)
        return None if best is None else best[1]

    npiv, status = 0, OPTIMAL
    try:
        solve_x()
        # 2. push
        for j in range(n):
            if stat[j] != INSIDE:
                continue
            if npiv >= maxp:
                status = MAX_ITER
                break
            _, d = solve_y()
            xj = xv[j]
            direction = 1 if d[j] < -told else -1 if d[j] > told else (1 if u[j] - xj < xj else -1)
            al = np.linalg.solve(B(), A[:, j])
            for _attempt in range(2):
                blk = primal_ratio(al, direction, 0.0, False)
                dist = u[j] - xj if direction > 0 else xj
                if blk is None and not np.isfinite(dist):
                    direction = -direction
                    continue
                if blk is not None and blk[1] < dist:
                    k, step, to_up = blk
                    xv[head] -= step * direction * al
                    xv[j] = xj + step * direction
                    v = head[k]
                    pivot(k, j, AT_UP if to_up else AT_LO, upper(v) if to_up else 0.0)
                    npiv += 1
                else:
                    xv[head] -= dist * direction * al
                    xv[j] = u[j] if direction > 0 else 0.0
                    stat[j] = AT_UP if direction > 0 else AT_LO
                break
        # 3. and 4.
        degen = 0
        for _round in range(4):
            if status != OPTIMAL:
                break
            solve_x()
            y, d = solve_y()
            pivoted = False
            while True:
                pv = primal_worst()
                bland = degen >= BLAND_AFTER
                infs = [(0.0 if bland else -dual_inf(j, d), j) for j in range(n) if dual_inf(j, d) > 0]
                q = min(infs)[1] if infs else None
                if pv is None and q is None:
                    break
                if pv is not None and q is not None:
                    status = NUMERICAL
                    break
                if npiv >= maxp:
                    status = MAX_ITER
                    break
                pivoted = True
                if q is not None:
                    direction = 1 if stat[q] == AT_LO else -1
                    al = np.linalg.solve(B(), A[:, q])
                    blk = primal_ratio(al, direction, tolp, bland)
                    if blk is None and not np.isfinite(u[q]):
                        status = NUMERICAL
                        break
                    if blk is None or u[q] <= blk[1]:
                        stat[q] = AT_UP if direction > 0 else AT_LO
                        xv[q] = u[q] if direction > 0 else 0.0
                        degen = 0
                    else:
                        k, theta, to_up = blk
                        v = head[k]
                        pivot(k, q, AT_UP if to_up else AT_LO, upper(v) if to_up else 0.0)
                        degen = degen + 1 if theta == 0.0 else 0
                else:
                    r = head.index(pv)
                    below = xv[pv] < 0.0
                    e, ratio = dual_ratio(row_alpha(r), d, -1 if below else 1, bland)
                    if e is None:
                        status = NUMERICAL
                        break
                    pivot(r, e, AT_LO if below else AT_UP, 0.0 if below else upper(pv))
                    degen = degen + 1 if ratio == 0.0 else 0
                npiv += 1
                solve_x()
                y, d = solve_y()
            if status != OPTIMAL:
                break
            for r in range(m):
                if head[r] < n:
                    continue
                if npiv >= maxp:
                    status = MAX_ITER
                    break
                alr = row_alpha(r)
                ep, rp_ = dual_ratio(alr, d, 1, False)
                en, rn_ = dual_ratio(alr, d, -1, False)
                e = en if ep is None else ep if en is None else (en if rn_ < rp_ else ep)
                if e is None:
                    continue
                pivot(r, e, AT_LO, 0.0)
                npiv += 1
                pivoted = True
                solve_x()
                y, d = solve_y()
            if status != OPTIMAL or not pivoted:
                break
        solve_x()
        y, d = solve_y()
        if status == OPTIMAL and (primal_worst() is not None or any(dual_inf(j, d) > 0 for j in range(n))):
            status = NUMERICAL
    except np.linalg.LinAlgError:
        status = NUMERICAL
        y, d = np.full(m, np.nan), np.full(n + m, np.nan)
    cs = np.where(stat[:n] == INSIDE, -1, stat[:n]).astype(np.int8)
    fixed = (u <= 0.0) & (cs != BASIC)
    cs[fixed] = np.where(d[:n][fixed] < 0.0, AT_UP, AT_LO)
    return dict(x=xv[:n].copy(), y=y, col_status=cs, row_basic=(stat[n:] == BASIC).astype(np.int8), status=status, pivots=npiv)
