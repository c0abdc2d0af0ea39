"""numpy f32 statement of the occupancy ESDF of a log-odds Octomap (DESIGN.md section 7, "Occupancy ESDF";
csrc/tslam_octo_esdf.cu).

Input: the known voxels of one submap as rows, `idx` int32[n,3] (centred indices) and `L` int32[n] (Q10 log-odds), as
OctoHandle.gather() returns them, plus l_occ, vs and D.  Nothing here knows about blocks or tiles.

    OCC  = L > l_occ,  FREE = the other known voxels; voxels without a row are UNKNOWN (neither sources nor targets)
    c1 = vs, c2 = f32(sqrt(2)) * vs, c3 = f32(sqrt(3)) * vs      (6-, 18-, 26-neighbours; f32 operations)
    FREE v starts at +D, OCC v at -D, and over its known 26-neighbours h:
        FREE v: E(v) = min(E(v), h OCC  ?  c : E(h) + c)
        OCC  v: E(v) = max(E(v), h FREE ? -c : E(h) - c)
    to the fixed point.

The iteration is Jacobi (every new value from the previous iterate), restricted after the first pass to the neighbours
of the voxels that changed; f32 min/+ is monotone, so the fixed point is unique and the schedule does not matter.
"""
import numpy as np

F = np.float32
_OFF = 1 << 20
OFFSETS = np.array([(dx, dy, dz) for dx in (-1, 0, 1) for dy in (-1, 0, 1) for dz in (-1, 0, 1) if (dx, dy, dz) != (0, 0, 0)],
                   np.int64)


def costs(vs):
    """(c1, c2, c3) as the kernels compute them: vs, sqrtf(2.0f) * vs, sqrtf(3.0f) * vs."""
    vs = F(vs)
    return vs, F(np.sqrt(F(2.0))) * vs, F(np.sqrt(F(3.0))) * vs


def pack(c):
    c = np.asarray(c, np.int64).reshape(-1, 3) + _OFF
    return (c[:, 0] << 42) | (c[:, 1] << 21) | c[:, 2]


def neighbours(idx):
    """int64[n,26]: row of each 26-neighbour (OFFSETS order), n where the neighbour has no row."""
    idx = np.asarray(idx, np.int64).reshape(-1, 3)
    n = idx.shape[0]
    keys = pack(idx)
    order = np.argsort(keys, kind="stable")
    sk = keys[order]
    nbr = np.full((n, len(OFFSETS)), n, np.int64)
    if n == 0:
        return nbr
    for k, off in enumerate(OFFSETS):
        q = pack(idx + off)
        p = np.minimum(np.searchsorted(sk, q), n - 1)
        hit = sk[p] == q
        nbr[hit, k] = order[p[hit]]
    return nbr


def esdf(idx, L, l_occ, vs, D, chunk=1 << 18):
    """-> E f32[n] in the row order of idx."""
    idx = np.asarray(idx, np.int64).reshape(-1, 3)
    L = np.asarray(L, np.int64).reshape(-1)
    n = idx.shape[0]
    D = F(D)
    occ = L > int(l_occ)
    E = np.where(occ, -D, D).astype(F)
    nbr = neighbours(idx)
    c1, c2, c3 = costs(vs)
    nz = np.abs(OFFSETS).sum(1)
    cost = np.where(nz == 1, c1, np.where(nz == 2, c2, c3)).astype(F)[None, :]
    occ_x = np.append(occ, False)      # row n: "no neighbour"
    has_x = np.append(np.ones(n, bool), False)
    active = np.arange(n)
    while active.size:
        Ex = np.append(E, F(0))
        new = np.empty(active.size, F)
        for s in range(0, active.size, chunk):
            a = active[s:s + chunk]
            h = nbr[a]
            hv, ho, hk = Ex[h], occ_x[h], has_x[h]
            vo = occ[a][:, None]
            with np.errstate(over="ignore", invalid="ignore"):
                cand_free = np.where(ho, cost, hv + cost)              # FREE v: from an OCC h the constant c
                cand_occ = np.where(~ho, -cost, hv - cost)             # OCC v: from a FREE h the constant -c
            lo = np.where(hk & ~vo, cand_free, F(np.inf)).min(1)
            hi = np.where(hk & vo, cand_occ, F(-np.inf)).max(1)
            cur = E[a]
            new[s:s + chunk] = np.where(occ[a], np.maximum(cur, hi), np.minimum(cur, lo))
        ch = new != E[active]
        changed = active[ch]
        E[changed] = new[ch]
        nxt = nbr[changed].reshape(-1)
        active = np.unique(nxt[nxt < n])
    return E
