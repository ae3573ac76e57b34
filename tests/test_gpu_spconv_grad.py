"""Backward of the sparse convs on the GPU, one operator at a time and end to end (SpMiddleFHD in train mode).

Bounds: the weight-gradient bounds are derived in tests/spconv_grad_model.py; the data gradient is the forward kernels with re-packed
weights, so it is held to the forward's bounds of tests/test_gpu_spconv_ops.py applied to those weights (fp32 rows kernel: (P Cin + 2) u
mag; cg: the accumulation term with G = 2 P Cp / 16 plus 2^-20 of the split magnitudes).
"""
import numpy as np
import pytest
import torch

from oracle.spconv_grad_ref import conv_backward_from_nbr, transpose_nbr
from spconv_grad_model import CG_C, U, WgradCase, pow2_scale_for_bound, ratio, spmiddle_train_ref
from test_gpu_spconv_ops import crafted_nbr

pytestmark = pytest.mark.gpu
NUM_SMS = 132


def _dev(a, dtype=torch.int32):
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda", dtype)


def _strided_nbr(n_out, n_in, kvol, seed):
    """a strided-like table: every (input row, offset) feeds at most one output row"""
    rng = np.random.default_rng(seed)
    nbr = np.full((n_out, kvol), -1, np.int64)
    for k in range(kvol):
        o = np.nonzero(rng.random(n_out) < 0.4)[0]
        nbr[o, k] = rng.permutation(n_in)[:len(o)] if len(o) <= n_in else rng.permutation(n_in)[np.arange(len(o)) % n_in]
        if len(o) > n_in:
            nbr[o[n_in:], k] = -1
    return nbr


def test_rulebook_transpose_is_exact():
    from sessd_b200 import ops
    for n_out, n_in, kvol, seed in ((1, 5, 27, 0), (129, 300, 27, 1), (5000, 4000, 27, 2), (777, 2000, 3, 3)):
        nbr = _strided_nbr(n_out, n_in, kvol, seed)
        max_out = n_out + 17
        full = np.concatenate([nbr, np.random.default_rng(seed).integers(0, n_in, (17, kvol))], 0)   # rows >= n ignored
        got = ops.rulebook_transpose(_dev(full), _dev([n_out]), max_out, n_in + 3).cpu().numpy()
        ref = np.full((n_in + 3, kvol), -1)
        ref[:n_in] = transpose_nbr(nbr, n_in)
        assert np.array_equal(got, ref)


def _ring_levels(batch=1, points=20000, seed=0):
    """the rulebooks of every strided level of a real frame (ring cloud) through the spconv modules: [(nbr, n_out, n_in)]"""
    import spconv
    from oracle import cpu as ocpu
    from sessd_b200 import synth
    from sessd_b200.runners import SPMIDDLE_LAYERS
    feats, coors = [], []
    for b in range(batch):
        v, c, n = ocpu.points_to_voxel(synth.ring_cloud(seed + b, points), synth.VOXEL_SIZE, synth.PC_RANGE, 5, 20000)
        coors.append(np.concatenate([np.full((len(c), 1), b, np.int32), c], 1))
        feats.append((v.sum(1) / n[:, None]).astype(np.float32))
    coors, feats = np.concatenate(coors), np.concatenate(feats)
    x = spconv.SparseConvTensor(torch.from_numpy(feats).cuda(), torch.from_numpy(coors).cuda(), [41, 1600, 1408], batch)
    out, cin = [], 4
    for kind, cout, ks, st, pd, key in SPMIDDLE_LAYERS:
        if kind != "subm":
            conv = spconv.SparseConv3d(cin, cout, ks, st, padding=list(pd), bias=False).cuda()
            y, nbr, n_out_t, cap = conv.rulebook(x)
            out.append((nbr, int(n_out_t.item()), int(x.indices.shape[0]), y))
            x = y
            x.features = torch.zeros((y.indices.shape[0], cout), device="cuda")
        cin = cout
    return out, coors, feats


def test_transpose_and_dense_grad_on_ring_levels():
    from sessd_b200 import ops
    levels, _c, _f = _ring_levels()
    assert len(levels) == 4
    for nbr, n_out, n_in, y in levels:
        got = ops.rulebook_transpose(nbr, _dev([n_out]), nbr.shape[0], n_in).cpu().numpy()
        assert np.array_equal(got, transpose_nbr(nbr.cpu().numpy()[:n_out], n_in))
    # dense() adjoint on the last level: every gathered value is the one dense() wrote there
    _nbr, n, _ni, y = levels[-1]
    d, h, w = y.spatial_shape
    c = 8
    grad = torch.randn((1, h, w, c * d), device="cuda")
    coors = y.indices.int().contiguous()
    got = ops.dense_grad_gather(grad, coors, _dev([n]), n + 5, ops.make_grid(1, y.spatial_shape), c,
                                torch.full((n + 5, c), -7.0, device="cuda")).cpu().numpy()
    q = coors.cpu().numpy().astype(np.int64)
    g = grad.cpu().numpy()
    ref = g[q[:, 0], q[:, 2], q[:, 3]].reshape(n, c, d)[np.arange(n), :, q[:, 1]]
    assert np.array_equal(got[:n], ref) and (got[n:] == -7.0).all()


def test_split_planes_bound_and_untouched_rows():
    from sessd_b200 import ops
    rng = np.random.default_rng(4)
    for n, c, cp in ((1, 32, 32), (1000, 64, 64), (300, 16, 32)):
        x = (rng.standard_normal((n + 9, c)) * np.exp2(rng.uniform(-10, 4, (n + 9, 1)))).astype(np.float32)
        xd = _dev(x, torch.float32)
        info = torch.zeros(2, device="cuda")
        ops.absmax_rows(xd, _dev([n]), n + 9, info[0:1])
        planes = torch.full((n + 9, 2 * cp), 3.0, dtype=torch.float16, device="cuda")
        ops.sparse_split_planes(xd, _dev([n]), n + 9, info, planes)
        s = float(info[1])
        amax = float(np.abs(x[:n]).max())
        assert float(info[0]) == amax and s == pow2_scale_for_bound(amax)
        p = planes.cpu().numpy().astype(np.float64)
        back = (p[:n, :c] + p[:n, cp:cp + c]) / s
        assert (np.abs(back - x[:n]) <= 2.0 ** -22 * amax).all()
        assert (p[:n, c:cp] == 0).all() and (p[:n, cp + c:] == 0).all() and (p[n:] == 3.0).all()


# ------------------------------------------------------------------------------------------------------------------ data gradient
@pytest.mark.parametrize("impl,cin,cout,subm", [("rows", 16, 16, True), ("rows", 16, 32, False), ("cg", 32, 32, True), ("cg", 32, 64, False),
                                                ("cg", 64, 64, True), ("cg", 64, 64, False)])
def test_dgrad_matches_fp64(impl, cin, cout, subm):
    """the data gradient through SparseConvFunction (forward kernel, re-packed weights, same / transposed table) vs conv_backward_from_nbr"""
    check_dgrad(impl, cin, cout, subm)


def check_dgrad(impl, cin, cout, subm, n_in=3000, n_out=2500):
    """test_dgrad_matches_fp64 on n_in input rows (and n_out output rows of a strided table)"""
    from sessd_b200 import sparse_grad
    rng = np.random.default_rng(cin + cout + subm)
    kvol = 27
    if subm:
        # a point-symmetric table: nbr[o, k] = i  <=>  nbr[i, K-1-k] = o
        nbr = np.full((n_in, kvol), -1, np.int64)
        for k in range(kvol // 2):
            o = rng.permutation(n_in)[:n_in // 3]
            i = rng.permutation(n_in)[:n_in // 3]
            nbr[o, k] = i
            nbr[i, kvol - 1 - k] = o
        nbr[:, kvol // 2] = np.arange(n_in)
        n_out = n_in
    else:
        nbr = _strided_nbr(n_out, n_in, kvol, cin)
    x = rng.standard_normal((n_in, cin)).astype(np.float32)
    w = (rng.standard_normal((3, 3, 3, cin, cout)) / np.sqrt(27 * cin)).astype(np.float32)
    g = rng.standard_normal((n_out, cout)).astype(np.float32)

    class _Rb(sparse_grad.ConvRulebook):
        def __init__(self):
            self.nbr, self.n_out_t, self.cap_out, self.n_out = _dev(nbr), _dev([n_out]), n_out, n_out
            self.n_in, self.n_in_t, self.cap_in, self.kvol, self.subm = n_in, _dev([n_in]), n_in, kvol, subm
            self._tiles = self._nbr_t = self._tiles_t = None

    xt = _dev(x, torch.float32).requires_grad_(True)
    wt = _dev(w, torch.float32).requires_grad_(True)
    out = sparse_grad.SparseConvFunction.apply(xt, wt, _Rb())
    assert sparse_grad.conv_impl(cin) == impl
    out.backward(_dev(g, torch.float32))
    gx_ref, _ = conv_backward_from_nbr(x, nbr, w.reshape(kvol, cin, cout), g)
    gx = xt.grad.cpu().numpy()
    ax, aw, ag = np.abs(x).astype(np.float64), np.abs(w.reshape(kvol, cin, cout)).astype(np.float64), np.abs(g).astype(np.float64)
    mag, _ = conv_backward_from_nbr(ax, nbr, aw, ag)
    P = np.zeros(n_in)
    for k in range(kvol):
        o = nbr[:, k] >= 0
        np.add.at(P, nbr[o, k], 1)
    if impl == "rows":
        tol = (P[:, None] * cout + 2) * U * mag
    else:
        gmax, wmax = float(ag.max()), aw.max(axis=(0, 2))               # per input channel c: the dgrad's output channel
        # split term: sum over pairs of (amax_g |w| + |g| wmax); accumulation term with G = 2 P Cout / 16
        sum_w, _ = conv_backward_from_nbr(np.ones_like(ax), nbr, aw, np.ones_like(ag))
        sum_g, _ = conv_backward_from_nbr(np.ones_like(ax), nbr, np.ones_like(aw), ag)
        tol = CG_C * 2.0 ** -23 * (2 * P[:, None] * cout / 16 + 2) * mag * 1.01 + 2.0 ** -20 * (gmax * sum_w + sum_g * wmax[None, :])
    r = ratio(gx, gx_ref, tol)
    print("dgrad %s (%d,%d) subm=%s ratio %.3g" % (impl, cin, cout, subm, r))
    assert r <= 1.0


# ------------------------------------------------------------------------------------------------------------------ weight gradient
def _wgrad_case(kind, cin, cout, kvol, seed):
    rng = np.random.default_rng(seed)
    if kind == "zero_one":            # offsets with 0 pairs and with exactly 1 pair
        n_out, n_in = 1000, 500
        nbr = crafted_nbr("full", n_out, kvol, n_in, seed)
        nbr[:, 0] = -1
        nbr[:, 1] = -1
        nbr[517, 1] = 3
    elif kind == "many_tiles":        # few offsets, items spanning many tiles
        n_out, n_in = 60000, 20000
        nbr = crafted_nbr("empty_tiles", n_out, kvol, n_in, seed)
    else:                             # more items than SMs, partial last tile
        n_out, n_in = 3 * NUM_SMS * 128 + 77, 5000
        nbr = crafted_nbr("flip", n_out, kvol, n_in, seed)
    max_out = n_out + 40
    full = np.concatenate([nbr, rng.integers(0, n_in, (40, kvol))], 0)
    x = rng.standard_normal((n_in, cin)).astype(np.float32)
    g = rng.standard_normal((max_out, cout)).astype(np.float32)
    return WgradCase(full, n_out, max_out, x, g)


def _run_wgrad(case, impl):
    from sessd_b200 import ops
    nbr = _dev(case.nbr)
    n = _dev([case.n_out])
    tiles = ops.rulebook_tile_lists(nbr, n, case.max_out, ops.alloc_tile_lists(case.max_out, case.kvol, "cuda"))
    x, g = _dev(case.x, torch.float32), _dev(case.g, torch.float32)
    if impl == "rows":
        return ops.spconv_wgrad_rows(x, g, tiles, n, case.max_out, case.kvol).cpu().numpy()
    xi, gi = torch.zeros(2, device="cuda"), torch.zeros(2, device="cuda")
    ops.absmax_rows(x, _dev([x.shape[0]]), x.shape[0], xi[0:1])
    ops.absmax_rows(g, n, case.max_out, gi[0:1])
    xp = ops.sparse_split_planes(x, _dev([x.shape[0]]), x.shape[0], xi, ops.alloc_planes(x.shape[0], case.cin, "cuda"))
    gp = ops.sparse_split_planes(g, n, case.max_out, gi, ops.alloc_planes(case.max_out, case.cout, "cuda"))
    return ops.spconv_wgrad_cg(xp, xi, gp, gi, tiles, n, case.max_out, case.kvol).cpu().numpy()


@pytest.mark.parametrize("impl,cin,cout", [("rows", 4, 16), ("rows", 16, 16), ("rows", 16, 32), ("cg", 32, 32), ("cg", 32, 64), ("cg", 64, 64)])
@pytest.mark.parametrize("kind,kvol", [("zero_one", 27), ("many_tiles", 3), ("many_items", 27)])
def test_wgrad_matches_emulation_and_fp64(impl, cin, cout, kind, kvol):
    from sessd_b200 import ops
    case = _wgrad_case(kind, cin, cout, kvol, cin * 7 + cout + kvol)
    assert ops.wgrad_items(case.max_out, kvol) == kvol * case.chunks
    if kind == "many_items":
        assert kvol * case.chunks > NUM_SMS
    got = _run_wgrad(case, impl)
    again = _run_wgrad(case, impl)
    assert got.tobytes() == again.tobytes(), "two runs differ"
    truth = case.truth()
    if impl == "rows":
        r = ratio(got, truth, case.tol_rows())
        print("wgrad rows %s (%d,%d) ratio %.3g" % (kind, cin, cout, r))
        assert r <= 1.0
    else:
        re, rf = ratio(got, case.emul(), case.tol_emul()), ratio(got, truth, case.tol_fp64())
        print("wgrad cg %s (%d,%d) ratio emul %.3g fp64 %.3g" % (kind, cin, cout, re, rf))
        assert re <= 1.0 and rf <= 1.0
    if kind == "zero_one":
        assert (got[0] == 0).all()


# ------------------------------------------------------------------------------------------------------------------ end to end
def test_spmiddle_train_forward_backward_matches_fp64():
    """SpMiddleFHD.train() on a 5k-point ring cloud, batch 2: dense output, every conv weight gradient and BN gamma / beta gradient within
    1e-4 of max |ref| of that tensor, running stats equal; the no-grad train-mode forward bitwise equal to the grad-mode one"""
    from det3d.models.backbones.scn import SpMiddleFHD
    from oracle import cpu as ocpu
    from sessd_b200 import synth
    feats, coors = [], []
    for b in range(2):
        v, c, n = ocpu.points_to_voxel(synth.ring_cloud(40 + b, 5000), synth.VOXEL_SIZE, synth.PC_RANGE, 5, 20000)
        coors.append(np.concatenate([np.full((len(c), 1), b, np.int32), c], 1))
        feats.append((v.sum(1) / n[:, None]).astype(np.float32))
    coors, feats = np.concatenate(coors), np.concatenate(feats)
    torch.manual_seed(0)
    m = SpMiddleFHD(num_input_features=4).cuda()
    with torch.no_grad():
        for mod in m.middle_conv:
            if isinstance(mod, torch.nn.BatchNorm1d):
                mod.weight.uniform_(0.5, 1.5)
                mod.bias.uniform_(-0.2, 0.2)
    # fp64 CPU restatement on copies of the parameters / running stats
    params = []
    for i in range(len(m.middle_conv) // 3):
        conv, bn = m.middle_conv[3 * i], m.middle_conv[3 * i + 1]
        params.append(dict(weight=conv.weight.detach().cpu().double().requires_grad_(True),
                           gamma=bn.weight.detach().cpu().double().requires_grad_(True), beta=bn.bias.detach().cpu().double().requires_grad_(True),
                           mean=bn.running_mean.detach().cpu().double().clone(), var=bn.running_var.detach().cpu().double().clone()))
    m.train()
    with torch.no_grad():
        m2 = SpMiddleFHD(num_input_features=4).cuda()
        m2.load_state_dict(m.state_dict())
        m2.train()
        d_nograd = m2(torch.from_numpy(feats).cuda(), torch.from_numpy(coors).cuda(), 2, [1408, 1600, 40])
    dense = m(torch.from_numpy(feats).cuda(), torch.from_numpy(coors).cuda(), 2, [1408, 1600, 40])
    assert tuple(dense.shape) == (2, 128, 200, 176)
    assert torch.equal(dense.detach(), d_nograd), "no-grad train-mode forward differs from the grad-mode forward"
    R = torch.randn(dense.shape, generator=torch.Generator().manual_seed(5), dtype=torch.float64)
    (dense * R.float().cuda()).sum().backward()
    ref = spmiddle_train_ref(torch.from_numpy(feats).double(), coors, 2, [1408, 1600, 40], params)
    (ref * R).sum().backward()

    def rel(got, want):
        got, want = got.detach().cpu().double(), want.detach().double()
        return float((got - want).abs().max() / max(float(want.abs().max()), 1e-30))

    trace = ["dense %.2e" % rel(dense, ref)]
    worst = rel(dense, ref)
    for i, p in enumerate(params):
        conv, bn = m.middle_conv[3 * i], m.middle_conv[3 * i + 1]
        errs = (rel(conv.weight.grad, p["weight"].grad), rel(bn.weight.grad, p["gamma"].grad), rel(bn.bias.grad, p["beta"].grad),
                rel(bn.running_mean, p["mean"]), rel(bn.running_var, p["var"]))
        trace.append("layer %d: gW %.2e  gamma %.2e  beta %.2e  mean %.2e  var %.2e" % ((i,) + errs))
        worst = max(worst, max(errs))
    print("\n".join(trace))
    assert worst <= 1e-4, "\n".join(trace)


def test_in_place_change_between_forward_and_backward_raises():
    """the conv Function keeps its weight, and on the fp32 layers its input, through save_for_backward: modifying them in place before
    backward is an error, not a silently wrong gradient (the tensor-core layers keep the input's planes, a copy made by the forward)"""
    from sessd_b200 import sparse_grad
    import spconv
    rng = np.random.default_rng(8)
    coors = np.unique(np.c_[np.zeros((400, 1)), rng.integers(0, 6, (400, 1)), rng.integers(0, 30, (400, 2))].astype(np.int32), axis=0)
    for cin, targets in ((16, ("input", "weight")), (32, ("weight",))):
        conv = spconv.SubMConv3d(cin, 32, 3, bias=False, indice_key="t").cuda()
        for target in targets:
            x = spconv.SparseConvTensor(torch.randn((len(coors), cin), device="cuda"), torch.from_numpy(coors).cuda(), [6, 30, 30], 1)
            feat = x.features.requires_grad_(target == "input")
            y, _rb = sparse_grad.sparse_conv(conv, x, {})
            with torch.no_grad():
                (feat if target == "input" else conv.weight).mul_(2.0)
            with pytest.raises(RuntimeError):
                y.features.sum().backward()
            conv.weight.grad = None
