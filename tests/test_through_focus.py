"""CPU: through-focus spot analysis (analyses.through_focus) without a device.

The plane selection, the default planes, the per-plane aberration formula and the sharded
gather of the [K*n_tiles, 16] sums.  The kernels themselves are compared with rt_trace_grid
plane by plane in test_gpu_through_focus.py."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from conftest import load_model
from rayoptics_b200 import _abi, table as T, engine as E, parallel as P, analyses as A
from rayoptics_b200.opticalspec import FocusRange

FOC = [0.0, -0.05, 0.02, -0.0, 0.125]


def test_default_planes_follow_the_focus_range():
    fr = FocusRange(focus_shift=0.03, defocus_range=0.2)
    got = A.focus_planes(fr, 7)
    # raytr/opticalspec.py FocusRange.get_focus: focus_shift + fr*defocus_range
    want = np.array([0.03 + f*0.2 for f in np.linspace(-1, 1, 7)])
    assert got.view(np.uint64).tolist() == want.view(np.uint64).tolist()
    assert got[3] == 0.03


def test_zero_defocus_range_without_foc_raises():
    opm = load_model('dblgauss')
    assert opm.optical_spec.defocus.defocus_range == 0
    with pytest.raises(ValueError, match='defocus_range'):
        A.through_focus(opm, 8)
    with pytest.raises(ValueError):
        A.focus_planes(FocusRange(0.1, 0.0), 5)


def test_best_plane_selection():
    foc = np.array([-0.2, -0.1, 0.0, 0.1])
    # [K=4, n_fields=2, n_wvls=3]
    rms = np.array([[[3., 1., 5.], [2., 2., 0.]],
                    [[2., 1., 4.], [2., 2., 0.]],
                    [[1., 1., 3.], [2., 2., 0.]],
                    [[2., 1., 2.], [2., 2., 0.]]])
    n_ok = np.full(rms.shape, 10.0)
    n_ok[:, 1, 2] = 0.0                    # no ray at the image: rms reads 0 there
    idx, best = A.best_focus(foc, rms, n_ok)
    assert idx.tolist() == [[2, 0, 3], [0, 0, -1]]          # ties: the first plane
    assert best[0].tolist() == [0.0, -0.2, 0.1] and best[1, :2].tolist() == [-0.2, -0.2]
    assert np.isnan(best[1, 2])
    nan_rms = rms.copy()
    nan_rms[0, 0, 0] = np.nan
    assert A.best_focus(foc, nan_rms, n_ok)[0][0, 0] == 2


def test_result_object_uses_spot_statistics_keys():
    k, nf, nw = 3, 2, 1
    s = np.zeros((k*nf*nw, 16))
    s[:, 0] = 4
    s[:, 7] = s[:, 8] = [4., 1., 9., 4., 1., 9.]            # rows (plane, field): field 0 least at plane 2
    stats = {key: np.asarray(v).reshape(k, nf, nw) for key, v in E.spot_statistics(s).items()}
    tf = A.ThroughFocus(np.array([0.0, 0.1, 0.2]), stats, np.zeros((k, nf, 2)), 8, nf, nw)
    assert tf.best_index.tolist() == [[2], [0]]
    assert tf.best_foc.tolist() == [[0.2], [0.0]]


def _oracle_grid(oracle, name='dblgauss', num=9):
    opm = load_model(name)
    descs, n_by_wvl, _ = T.describe_model(opm.seq_model)
    spec = E.grid_spec_for_model(opm, num)
    opts = _abi.make_opts(first_surf=1, last_surf=len(descs) - 2, check_apertures=True)
    r = oracle.trace_grid(spec.c_spec(), descs, n_by_wvl, 0, spec.n_rays, opts)
    return opm, spec, r


def test_per_plane_formula_matches_focus_pupil_coords(oracle):
    """The kernels evaluate plane k as the single-focus epilogue with foc -> foc[k]; the oracle's
    restatement of that epilogue equals the reference's focus_pupil_coords arithmetic
    (analyses._refocused) bit for bit, for the rays and for the defocused chief-ray point."""
    opm, spec, r = _oracle_grid(oracle)
    ok = r['status'] == 0
    assert ok.sum() > 100
    p, d = r['last'][0:3][:, ok], r['last'][3:6][:, ok]
    chief_p, chief_d = p[:, 0], d[:, 0]                     # any ray will do as the chief ray
    for foc in FOC + [opm.optical_spec.defocus.focus_shift]:
        dist = foc/chief_d[2]
        ref = chief_p + dist*chief_d                        # calculate_reference_sphere's image_pt
        ax, ay = oracle.transverse_abr(p[0], p[1], d[0], d[1], d[2], foc, ref[0], ref[1])
        want = np.array([A._refocused(([(p[:, i], d[:, i])],), foc, ref)[:2] for i in range(p.shape[1])])
        assert ax.view(np.uint64).tolist() == want[:, 0].view(np.uint64).tolist(), foc
        assert ay.view(np.uint64).tolist() == want[:, 1].view(np.uint64).tolist(), foc


def focus_sums(oracle, spec, r, ray_begin, foc, ref):
    """[K, n_tiles, 16] partial sums of oracle rays starting at ray_begin, plane k referred to
    ref[k][field]."""
    out = np.zeros((len(foc), spec.n_tiles, 16))
    out[:, :, 10] = out[:, :, 12] = np.inf
    out[:, :, 11] = out[:, :, 13] = -np.inf
    n = r['status'].shape[0]
    tiles = (ray_begin + np.arange(n))//spec.rays_per_tile
    last = r['last']
    for k, f in enumerate(foc):
        for t in np.unique(tiles):
            m = tiles == t
            st = r['status'][m]
            okm = st == 0
            fi = t//spec.n_wvls
            ax, ay = oracle.transverse_abr(last[0][m][okm], last[1][m][okm], last[3][m][okm], last[4][m][okm],
                                           last[5][m][okm], f, ref[k][fi][0], ref[k][fi][1])
            out[k, t, 0:5] = [okm.sum(), (st == 1).sum(), (st == 2).sum(), (st == 3).sum(), (st > 3).sum()]
            if okm.any():
                out[k, t, 5:10] = [ax.sum(), ay.sum(), (ax*ax).sum(), (ay*ay).sum(), (ax*ay).sum()]
                out[k, t, 10:14] = [ax.min(), ax.max(), ay.min(), ay.max()]
                out[k, t, 14] = r['op'][m][okm].sum()
    return out


def _setup():
    from oracle import rt_oracle
    opm = load_model('dblgauss')
    descs, n_by_wvl, _ = T.describe_model(opm.seq_model)
    spec = E.grid_spec_for_model(opm, 24)
    opts = _abi.make_opts(first_surf=1, last_surf=len(descs) - 2, check_apertures=True)
    ref = np.stack([np.full((spec.n_fields, 2), 0.01*k) for k in range(len(FOC))])
    return rt_oracle, spec, descs, n_by_wvl, opts, ref


def worker(rank, world, port, q):
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    try:
        oracle, spec, descs, n_by_wvl, opts, ref = _setup()
        c0, c1 = P.shard_chunks(spec.n_chunks, rank, world)
        r0, r1 = spec.first_ray_of_chunk(c0), spec.first_ray_of_chunk(c1)
        r = oracle.trace_grid(spec.c_spec(), descs, n_by_wvl, r0, r1, opts)
        part = torch.from_numpy(focus_sums(oracle, spec, r, r0, FOC, ref))
        # as through_focus: the flattened [K*n_tiles, 16] block in one collective
        comb = P.gather_summaries(part.reshape(-1, 16)).reshape(part.shape)
        q.put((rank, r1 - r0, comb.numpy()))
    finally:
        dist.destroy_process_group()


def test_sharded_focus_summaries_world2():
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        port = s.getsockname()[1]
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    procs = [ctx.Process(target=worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = [q.get(timeout=120) for _ in procs]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    oracle, spec, descs, n_by_wvl, opts, ref = _setup()
    whole = focus_sums(oracle, spec, oracle.trace_grid(spec.c_spec(), descs, n_by_wvl, 0, spec.n_rays, opts),
                       0, FOC, ref)
    assert sum(g[1] for g in got) == spec.n_rays
    for rank, _, comb in got:
        assert comb.shape == (len(FOC), spec.n_tiles, 16)
        assert np.array_equal(comb[..., 0:5], whole[..., 0:5])
        assert np.array_equal(comb[..., 10:14], whole[..., 10:14])
        np.testing.assert_allclose(comb[..., 5:10], whole[..., 5:10], rtol=1e-11, atol=1e-12)
        np.testing.assert_allclose(comb[..., 14], whole[..., 14], rtol=1e-12)
    assert not np.array_equal(whole[0, :, 5], whole[-1, :, 5])     # the planes differ
