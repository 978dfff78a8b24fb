"""Host-side scene input for codimensional components: tet meshes plus kinematic triangle (.obj, codimension 2), segment (.seg,
codimension 1) and point (.pt, codimension 0) shapes, assembled into the arrays the reference's Mesh<3> builds for them
(main.cpp:948-1010 loading, Mesh.cpp:273-411 masses, :470-515 vNeighbor and SFEdges, :904-928 SVI).

The result is a Mesh whose arrays go to the C ABI unchanged: SVI / SFEdges / SF / vCoDim to ipcgpu_set_surface, mass and dbc to
ipcgpu_set_mesh, csr_pattern() to ipcgpu_set_csr.  Codimensional components carry no tets and so no elasticity (the reference has none).
"""
import os

import numpy as np

from . import mesh as M


def read_obj(path):
    """igl::readOBJ's vertices and triangles (1-based `f a b c`, `a/b/c` index groups allowed)."""
    V, F = [], []
    with open(path) as f:
        for line in f:
            tok = line.split()
            if not tok:
                continue
            if tok[0] == "v":
                V.append([float(x) for x in tok[1:4]])
            elif tok[0] == "f":
                F.append([int(x.split("/")[0]) - 1 for x in tok[1:4]])
    return np.asarray(V, dtype=np.float64).reshape(-1, 3), np.asarray(F, dtype=np.int32).reshape(-1, 3)


def obj_edges(F):
    """main.cpp:968-992: the edges of an .obj's triangles, (a, b) kept unless (b, a) was inserted before, in std::set order."""
    return M.surface_edges(np.asarray(F, dtype=np.int32).reshape(-1, 3)) if len(F) else np.zeros((0, 2), dtype=np.int32)


def read_seg(path):
    """IglUtils::readSEG (`v x y z`, 1-based `s a b`); a missing file falls back to the edges of the same-stem .obj (main.cpp:962-992)."""
    if not os.path.exists(path):
        V, F = read_obj(os.path.splitext(path)[0] + ".obj")
        return V, obj_edges(F)
    V, E = [], []
    with open(path) as f:
        for line in f:
            tok = line.split()
            if not tok:
                continue
            if tok[0] == "v":
                V.append([float(x) for x in tok[1:4]])
            elif tok[0] == "s":
                E.append([int(tok[1]) - 1, int(tok[2]) - 1])
    return np.asarray(V, dtype=np.float64).reshape(-1, 3), np.asarray(E, dtype=np.int32).reshape(-1, 2)


def read_pt(path):
    """main.cpp:996-1004: the vertices of the .pt file read as an .obj, or of the same-stem .obj when it is missing."""
    if not os.path.exists(path):
        path = os.path.splitext(path)[0] + ".obj"
    return read_obj(path)[0]


def read_shape(path):
    """(codimension, V, primitives) of a shape file by suffix: .obj triangles (2), .seg segments (1), .pt points (0)."""
    ext = os.path.splitext(path)[1]
    if ext == ".obj":
        V, F = read_obj(path)
        return 2, V, F
    if ext == ".seg":
        V, E = read_seg(path)
        return 1, V, E
    if ext == ".pt":
        return 0, read_pt(path), None
    raise ValueError(f"unsupported codimensional shape file: {path}")


def _voronoi_tri_mass(V, F):
    """Mesh.cpp:311-395 (igl::massmatrix VORONOI per triangle corner, times the triangle's mean edge length / 3): (m, 3) corner masses."""
    x0, x1, x2 = V[F[:, 0]], V[F[:, 1]], V[F[:, 2]]
    l = np.stack([np.linalg.norm(x1 - x2, axis=1), np.linalg.norm(x2 - x0, axis=1), np.linalg.norm(x0 - x1, axis=1)], axis=1)
    ls = -np.sort(-l, axis=1)  # igl::doublearea from edge lengths: Kahan's stable Heron on the sorted lengths, 0 where it turns negative
    a, b, c = ls[:, 0], ls[:, 1], ls[:, 2]
    dblA = 2.0 * 0.25 * np.sqrt(np.maximum((a + (b + c)) * (c - (a - b)) * (c + (a - b)) * (a + (b - c)), 0.0))
    cosines = np.stack([(l[:, 2] ** 2 + l[:, 1] ** 2 - l[:, 0] ** 2) / (l[:, 1] * l[:, 2] * 2.0),
                        (l[:, 0] ** 2 + l[:, 2] ** 2 - l[:, 1] ** 2) / (l[:, 2] * l[:, 0] * 2.0),
                        (l[:, 1] ** 2 + l[:, 0] ** 2 - l[:, 2] ** 2) / (l[:, 0] * l[:, 1] * 2.0)], axis=1)
    bary = cosines * l
    bary = bary / bary.sum(1)[:, None]
    partial = bary * (dblA * 0.5)[:, None]
    quads = np.stack([(partial[:, 1] + partial[:, 2]) * 0.5, (partial[:, 2] + partial[:, 0]) * 0.5, (partial[:, 0] + partial[:, 1]) * 0.5], axis=1)
    for k in range(3):  # an obtuse corner k: a quarter of the area to it, an eighth to the others
        obt = cosines[:, k] < 0
        quads[obt] = np.outer(dblA[obt], [0.125, 0.125, 0.125])
        quads[obt, k] = 0.25 * dblA[obt]
    return quads * (l.mean(1) / 3.0)[:, None]


class CodimMesh(M.Mesh):
    """A Mesh with codimensional components.  Extra members, as the reference's Mesh<3> holds them:
    componentNodeRange / componentCoDim (per component), CE (codimension-1 segments), and SF with the codimension-2 triangles appended
    in component order."""

    def neighbor_pairs(self, extra_pairs=None):
        """vNeighbor (Mesh.cpp:470-493): tet edges, triangle edges and segments (SFEdges holds the last two) (+ contact pairs)."""
        pairs = self.SFEdges if extra_pairs is None or not len(extra_pairs) else np.concatenate([self.SFEdges, np.asarray(extra_pairs).reshape(-1, 2)])
        return super().neighbor_pairs(pairs)


def codim_scene(components, YM=1e5, PR=0.4, density=1000.0, energy=0):
    """Assemble a scene from components in the order the reference's `shapes` lines list them.  Each component is a dict with
    `codim` (3, 2, 1 or 0) and `V` (n, 3) already placed (scenes.shape_transform), plus `T` (tets; optional `SF`) for codimension 3,
    `F` for 2, `E` for 1; `dbc=True` flags every vertex of the component Dirichlet (a scripted component).  At least one tet component is
    needed (the point mass is the tet vertices' mean)."""
    Vs, Ts, SFs, CEs, cod, dbc, rng = [], [], [], [], [], [], [0]
    off = 0
    for c in components:
        V = np.asarray(c["V"], dtype=np.float64).reshape(-1, 3)
        k = int(c["codim"])
        if k == 3:
            T = np.asarray(c["T"], dtype=np.int32).reshape(-1, 4)
            SF = c.get("SF")
            SF = M.boundary_faces(T) if SF is None or len(SF) == 0 else np.asarray(SF, dtype=np.int32).reshape(-1, 3)
            Ts.append(T + off)
            SFs.append(SF + off)
        elif k == 2:
            SFs.append(np.asarray(c["F"], dtype=np.int32).reshape(-1, 3) + off)
        elif k == 1:
            CEs.append(np.asarray(c["E"], dtype=np.int32).reshape(-1, 2) + off)
        elif k != 0:
            raise ValueError("codimension must be 0, 1, 2 or 3")
        Vs.append(V)
        cod.append(np.full(len(V), k, dtype=np.int32))
        dbc.append(np.full(len(V), 1 if c.get("dbc") else 0, dtype=np.uint8))
        off += len(V)
        rng.append(off)
    if not Ts:
        raise ValueError("a codimensional scene needs at least one tet component")
    V = np.concatenate(Vs)
    T = np.concatenate(Ts)
    SF = np.concatenate(SFs).astype(np.int32)
    CE = np.concatenate(CEs).astype(np.int32) if CEs else np.zeros((0, 2), dtype=np.int32)
    m = CodimMesh(V, T, YM=YM, PR=PR, density=density, energy=energy, SF=SF)
    m.componentNodeRange = np.asarray(rng, dtype=np.int64)
    m.componentCoDim = np.asarray([int(c["codim"]) for c in components], dtype=np.int32)
    m.CE = CE
    m.vCoDim = np.concatenate(cod)
    m.dbc = np.concatenate(dbc)
    # SFEdges (Mesh.cpp:495-515): the triangles' edges in std::set order, then CE
    m.SFEdges = np.concatenate([M.surface_edges(SF), CE]).astype(np.int32)
    # SVI (Mesh.cpp:904-928): every vertex of SF or CE and every vertex without a neighbour, ascending
    on = np.zeros(m.nV, dtype=bool)
    on[SF.ravel()] = True
    on[CE.ravel()] = True
    has_nbr = np.zeros(m.nV, dtype=bool)
    has_nbr[T.ravel()] = True
    has_nbr[SF.ravel()] = True
    has_nbr[CE.ravel()] = True
    m.SVI = np.flatnonzero(on | ~has_nbr).astype(np.int32)
    # masses (Mesh.cpp:273-411): tets vol / 4 (the Mesh constructor), triangles Voronoi, segment ends l^3 pi / 12, all times density;
    # points the mean mass of the tet components' vertices, after the density scaling
    for c, lo in zip(components, rng[:-1]):
        if int(c["codim"]) == 2 and len(c["F"]):
            F = np.asarray(c["F"], dtype=np.int64).reshape(-1, 3) + lo
            np.add.at(m.mass, F.T.ravel(), density * _voronoi_tri_mass(V, F).T.ravel())
        elif int(c["codim"]) == 1 and len(c["E"]):
            E = np.asarray(c["E"], dtype=np.int64).reshape(-1, 2) + lo
            l = np.linalg.norm(V[E[:, 0]] - V[E[:, 1]], axis=1)
            np.add.at(m.mass, E.T.ravel(), density * np.tile(l ** 3 * np.pi / 12.0, 2))
    tet_v = np.concatenate([np.arange(rng[i], rng[i + 1]) for i, c in enumerate(components) if int(c["codim"]) == 3])
    avg = float(m.mass[tet_v].mean()) if len(tet_v) else 0.0
    m.mass[m.vCoDim == 0] = avg
    m.bbox_diag2 = float(((m.V_rest.max(0) - m.V_rest.min(0)) ** 2).sum())
    m._nbr = None
    return m


def component_ends(m):
    """(vertex_end, tet_end): the cumulative compVAccSize / compFAccSize of ipcgpu_set_components from componentNodeRange.  A tet belongs
    to the component of its first vertex (codim_scene appends the tets in component order); codimensional components add no tet."""
    rng = np.asarray(m.componentNodeRange, dtype=np.int64)
    comp_of_tet = np.searchsorted(rng, np.asarray(m.T)[:, 0], side="right") - 1
    tets = np.bincount(comp_of_tet, minlength=len(rng) - 1)
    return rng[1:].astype(np.int32), np.cumsum(tets).astype(np.int32)
