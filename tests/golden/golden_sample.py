"""Fixed, seeded samples of large fixture arrays, so that every fixture file stays under 1 MB.

A sampled array is stored as three entries: `<key>#i` (flat indices), `<key>#v` (the values there) and `<key>#shape`.  The
entries are drawn per group -- one group per section of a record (a field of a layout, on one grid point of one OCP) -- so
that every section of every record is covered: a fraction `frac` of its nonzero entries (at least `k_min`) and up to `k_z`
of its zero entries.  `restore` puts the sample into a copy of the array under test, so that comparing the two compares
exactly the sampled entries.  Arrays stored whole (`<key>`) are returned as they are.
"""
import math

import numpy as np


def layout_bounds(layout, prefix, stride):
    """[offset, next offset) of every field `<prefix>*` of a record layout (rbt_layout, rbt_stage_layout, ...)."""
    offs = sorted({v for k, v in vars(layout).items() if k.startswith(prefix) and isinstance(v, int)
                   and not k.endswith(("stride", "size")) and 0 <= v < stride})
    return list(zip(offs, offs[1:] + [stride]))


def groups(a, bounds=None):
    """Group id of every entry of `a` (records along all axes but the last): its record, and its section if `bounds`."""
    rec = np.arange(a.size // a.shape[-1]).reshape(a.shape[:-1] + (1,))
    if bounds is None:
        return np.broadcast_to(rec, a.shape)
    col = np.full(a.shape[-1], len(bounds))  # entries outside every section (padding) form a section of their own
    for n, (o, e) in enumerate(bounds):
        col[o:e] = n
    return rec * (len(bounds) + 1) + col


def sample(a, grp, seed, frac, k_min, k_z):
    """frac / k_min / k_z: one value for all groups, or a tuple indexed by group id."""
    rng = np.random.default_rng(seed)
    flat, gf = a.reshape(-1), np.asarray(grp).reshape(-1)
    pick = lambda v, g: v[g] if isinstance(v, tuple) else v  # noqa: E731
    idx = []
    for g in np.unique(gf):
        pos = np.flatnonzero(gf == g)
        nz, z = pos[flat[pos] != 0.0], pos[flat[pos] == 0.0]
        kn = min(nz.size, max(pick(k_min, g), math.ceil(pick(frac, g) * nz.size)))
        idx.append(rng.choice(nz, kn, replace=False))
        idx.append(rng.choice(z, min(pick(k_z, g), z.size), replace=False))
    idx = np.sort(np.concatenate(idx)).astype(np.int32)
    return {"i": idx, "v": flat[idx], "shape": np.array(a.shape)}


def put(out, key, a, grp=None, seed=0, frac=0.0, k_min=12, k_z=2):
    """Stores a seeded sample of `a` under `key` in the dict `out` (grp: group ids, default one group per record)."""
    for f, v in sample(a, groups(a) if grp is None else grp, seed, frac, k_min, k_z).items():
        out[f"{key}#{f}"] = v


def restore(G, key, base):
    """The reference array `key` of the fixture G: stored whole, or `base` (the array under test) with the sample put in."""
    if key in G:
        return np.array(G[key])
    assert tuple(G[f"{key}#shape"]) == np.shape(base), key
    out = np.array(base, dtype=np.float64, copy=True)
    out.reshape(-1)[G[f"{key}#i"]] = G[f"{key}#v"]
    return out


def load(path):
    """The fixture as a dict (name -> array)."""
    with np.load(path) as z:
        return {k: z[k] for k in z.files}
