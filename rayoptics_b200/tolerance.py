"""Toleranced parameters and the prescriptions of perturbed systems.

A ``Tolerance(kind, index, delta)`` is one parameter with the symmetric limit ``+-delta``; a
*change* is ``(tolerance, d)`` with the value ``d`` actually applied.  Two routes build a perturbed
system:

* ``perturbed_model(opt_model, changes)``, the truth path: a deep copy of the model with the
  changes applied and ``seq_model.update_model()`` run, which recomputes the indices, ``z_dir``
  and the interface transforms.  Apertures, vignetting, aim points, pupil and paraxial data stay
  nominal: the analysis is a sensitivity with the nominal mechanics and aim, without re-aiming.
* ``perturbed_descriptors(descs, n_by_wvl, changes, seq_model)``, the fast path: a copy of the
  nominal surface table with only the touched entries recomputed; the transforms come from the
  model's own ``forward_transform`` and ``DecenterData``.  Its bytes equal
  ``describe_model(perturbed_model(...).seq_model)``.

Kinds (``s``: an interface, 1 <= s <= n_ifc - 2; ``g``: a gap, 1 <= g <= n_gaps - 1):
``'radius'`` (r = 1/cv, cv' = 1/(r + d); a plane is refused), ``'conic'`` (cc' = cc + d,
ec' = cc' + 1; a Spherical profile becomes a Conic), ``'thickness'`` (gap g), ``'index'`` (every
wavelength's index of the medium after interface s, + d rounded once), ``'decenter_x'``,
``'decenter_y'`` (system units) and ``'tilt_x'``, ``'tilt_y'`` (degrees: alpha, beta) of
interface s, added to its ``DecenterData`` (``'dec and return'`` where it has none).
"""
from __future__ import annotations

import copy
import ctypes as C
import types
from dataclasses import dataclass

import numpy as np

from . import model as M
from ._abi import PROFILE_IDS
from .table import profile_fields, set_transform

KINDS = ('radius', 'conic', 'thickness', 'index', 'decenter_x', 'decenter_y', 'tilt_x', 'tilt_y')
_PROFILE_KINDS = ('radius', 'conic')
_DECENTER_KINDS = {'decenter_x': ('dec', 0), 'decenter_y': ('dec', 1), 'tilt_x': ('euler', 0),
                   'tilt_y': ('euler', 1)}


@dataclass(frozen=True)
class Tolerance:
    """One toleranced parameter: ``kind`` (``KINDS``), the interface or gap ``index`` it acts on,
    and the symmetric limit ``+-delta``."""
    kind: str
    index: int
    delta: float


def check(sm, tol):
    """ValueError unless ``tol`` can be applied to the sequential model ``sm``"""
    n_ifc = len(sm.ifcs)
    if tol.kind not in KINDS:
        raise ValueError(f'unknown tolerance kind {tol.kind!r}')
    i = int(tol.index)
    if tol.kind == 'thickness':
        if not 1 <= i <= len(sm.gaps) - 1:
            raise ValueError(f'thickness tolerance on gap {i}: gaps 1 .. {len(sm.gaps) - 1} only')
    elif not 1 <= i <= n_ifc - 2:
        raise ValueError(f'{tol.kind} tolerance on interface {i}: interfaces 1 .. {n_ifc - 2} only')
    if tol.kind in _PROFILE_KINDS:
        prof = getattr(sm.ifcs[i], 'profile', None)
        if prof is None or type(sm.ifcs[i]).__name__ == 'ThinLens':
            raise ValueError(f'{tol.kind} tolerance on interface {i}, which has no profile')
        if tol.kind == 'radius' and prof.cv == 0.0:
            raise ValueError(f'radius tolerance on the plane interface {i}')
    if (tol.kind == 'thickness' or tol.kind in _DECENTER_KINDS) and sm._tfrms_given is not None:
        raise ValueError(f'{tol.kind} tolerance on a model whose transforms were given explicitly')


def _new_profile(prof, kind, d):
    """the perturbed profile (a new object; ``prof`` is not changed)"""
    if kind == 'radius':
        p = copy.copy(prof)
        p.cv = 1.0/(1.0/prof.cv + d)
        return p
    name = type(prof).__name__
    if name == 'Spherical':
        return M.Conic(c=prof.cv, cc=0.0 + d)
    p = copy.copy(prof)
    cc = prof.cc + d
    if name == 'RadialPolynomial':     # stores ec, cc is derived
        p.ec = cc + 1.0
    else:
        p.cc = cc
    return p


def _new_decenter(ifc, kind, d):
    """the perturbed DecenterData of ``ifc`` (a new object)"""
    old = getattr(ifc, 'decenter', None)
    dd = copy.deepcopy(old) if old is not None else M.DecenterData('dec and return')
    attr, c = _DECENTER_KINDS[kind]
    getattr(dd, attr)[c] += d
    dd.update()
    return dd


class _IndexShift(M.Medium):
    """a medium whose index is another's + d (rounded once)"""

    def __init__(self, base, d):
        self.base, self.d = base, d

    def rindex(self, wvl):
        return self.base.rindex(wvl) + self.d


def _apply(sm, tol, d):
    i = int(tol.index)
    if tol.kind in _PROFILE_KINDS:
        sm.ifcs[i].profile = _new_profile(sm.ifcs[i].profile, tol.kind, d)
    elif tol.kind == 'thickness':
        sm.gaps[i].thi += d
    elif tol.kind == 'index':
        sm.gaps[i].medium = _IndexShift(sm.gaps[i].medium, d)
    else:
        sm.ifcs[i].decenter = _new_decenter(sm.ifcs[i], tol.kind, d)


def perturbed_model(opt_model, changes):
    """A deep copy of ``opt_model`` with every ``(tolerance, d)`` of ``changes`` applied, in order,
    and ``seq_model.update_model()`` run.  Apertures, vignetting, aim points, pupil and paraxial
    data stay nominal (no re-aiming)."""
    sm0 = opt_model.seq_model
    for tol, _ in changes:
        check(sm0, tol)
    memo = {}
    cached = getattr(sm0, '_b200_table', None)
    if cached is not None:             # the device table handle is not copied: the copy builds its own
        memo[id(cached)] = None
    opm = copy.deepcopy(opt_model, memo)
    sm = opm.seq_model
    for tol, d in changes:
        _apply(sm, tol, float(d))
    sm.update_model()
    return opm


def perturbed_descriptors(descs, n_by_wvl, changes, seq_model):
    """``(descs', n_by_wvl')``: the nominal surface table of ``seq_model`` (``describe_model``'s
    ``descs``, ``n_by_wvl``) with ``changes`` applied to the touched entries only -- cv, cc, ec,
    profile; the index column of the medium; the transforms of the interfaces before and after the
    change.  Bytes equal ``describe_model(perturbed_model(...).seq_model)``."""
    sm = seq_model
    n_ifc = len(descs)
    out = (type(descs[0])*n_ifc)()
    C.memmove(out, descs, C.sizeof(out))
    nb = np.array(n_by_wvl, dtype=np.float64, copy=True)
    profiles, decenters, thi, shifts = {}, {}, {}, {}
    for tol, d in changes:
        check(sm, tol)
        d, i = float(d), int(tol.index)
        if tol.kind in _PROFILE_KINDS:
            profiles[i] = _new_profile(profiles.get(i, sm.ifcs[i].profile), tol.kind, d)
        elif tol.kind == 'thickness':
            thi[i] = thi.get(i, sm.gaps[i].thi) + d
        elif tol.kind == 'index':
            shifts.setdefault(i, []).append(d)
        else:
            ifc = types.SimpleNamespace(decenter=decenters.get(i, getattr(sm.ifcs[i], 'decenter', None)))
            decenters[i] = _new_decenter(ifc, tol.kind, d)
    for i, p in profiles.items():
        pname = type(p).__name__
        out[i].profile = PROFILE_IDS[pname]
        out[i].cv, out[i].cc, out[i].ec = profile_fields(p, pname)
    if shifts:
        wvls = list(sm.wvlns)
        for i, ds in shifts.items():
            med = sm.gaps[i].medium
            for dd in ds:
                med = _IndexShift(med, dd)
            col = [med.rindex(w) for w in wvls]
            nb[:, i] = col
            if i + 1 == n_ifc - 1:         # the image interface has no gap: it repeats the last index
                nb[:, i + 1] = col
    touched = set(thi) | {j for i in decenters for j in (i - 1, i)}
    if touched:
        def ifc(j):
            return types.SimpleNamespace(decenter=decenters[j]) if j in decenters else sm.ifcs[j]
        for j in sorted(touched):
            r, t = M.forward_transform(ifc(j), thi.get(j, sm.gaps[j].thi), ifc(j + 1))
            set_transform(out[j], (r.transpose(), t))
    return out, np.ascontiguousarray(nb)
