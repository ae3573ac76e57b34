"""Rulebook (bit-exact vs the CPU restatement, canonical order) and sparse conv features (<= 1e-4 rel vs an fp64 oracle)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _voxels(cloud):
    from oracle import cpu as ocpu
    from sessd_b200 import synth
    v, c, n = ocpu.points_to_voxel(cloud, synth.VOXEL_SIZE, synth.PC_RANGE, 5, 20000)
    return v, np.concatenate([np.zeros((len(c), 1), np.int32), c], 1).astype(np.int32), n


def _two_frame_coors():
    from sessd_b200 import synth
    _, c0, _ = _voxels(synth.ring_cloud(3, 6000))
    _, c1, _ = _voxels(synth.uniform_cloud(4, 3000))
    c1[:, 0] = 1
    return np.concatenate([c0, c1], 0)


def test_subm_rulebook_hash_and_pairs_bit_exact():
    from oracle import spconv_ref as S
    from sessd_b200 import ops
    coors = _two_frame_coors()
    n = len(coors)
    shape = (41, 1600, 1408)
    grid = ops.make_grid(2, shape)
    cap = n + 100
    d_coors = torch.zeros((cap, 4), dtype=torch.int32, device="cuda")
    d_coors[:n] = torch.from_numpy(coors).cuda()
    d_n = torch.tensor([n], dtype=torch.int32, device="cuda")
    table = ops.hash_build(d_coors, d_n, cap, grid)
    nbr = ops.subm_rulebook(d_coors, d_n, cap, grid, (3, 3, 3), 0, table)
    ref = S.neighbor_table(coors, shape, coors, (3, 3, 3), (1, 1, 1), (1, 1, 1))
    got = nbr[:n].cpu().numpy()
    assert np.array_equal(got, ref)
    # canonical spconv pairs: per offset sorted by output index
    pin, pout, num = ops.rulebook_pairs(nbr, d_n, cap, 27)
    pairs = S.pairs_from_nbr(ref)
    num = num.cpu().numpy()
    for k in range(27):
        assert num[k] == len(pairs[k][0])
        assert np.array_equal(pin[k, : num[k]].cpu().numpy(), pairs[k][0])
        assert np.array_equal(pout[k, : num[k]].cpu().numpy(), pairs[k][1])
    assert int(num[13]) == n   # centre offset: every voxel pairs with itself


def test_strided_chain_rulebooks_bit_exact():
    """The 4 strided + 3 SubM(bitmap-indexed) rulebooks of SpMiddleFHD on a 2-frame batch."""
    from oracle import spconv_ref as S
    from sessd_b200 import ops
    from sessd_b200.runners import SpMiddleRunner
    coors = _two_frame_coors()
    n = len(coors)
    r = SpMiddleRunner(2, n + 50, device="cuda")
    layers, _, _ = _weights()
    r.load_weights(layers)
    d_coors = torch.zeros((n + 50, 4), dtype=torch.int32, device="cuda")
    d_coors[:n] = torch.from_numpy(coors).cuda()
    feat = torch.randn((n + 50, 4), device="cuda")
    r.forward(feat, d_coors, torch.tensor([n], dtype=torch.int32, device="cuda"))
    torch.cuda.synchronize()
    assert int(r.status.item()) == 0
    cur, shape = coors, (41, 1600, 1408)
    lvl = 0
    seen = set()
    for p in r.plan:
        if p["kind"] == "subm":
            if p["key"] in seen:
                continue
            seen.add(p["key"])
            ref = S.neighbor_table(cur, shape, cur, p["ks"], (1, 1, 1), (1, 1, 1))
            assert np.array_equal(p["nbr"][: len(cur)].cpu().numpy(), ref), p["key"]
        else:
            oc, oshape = S.strided_out_coors(cur, shape, p["ks"], p["st"], p["pd"])
            lv = r.levels[lvl + 1]
            assert int(lv["n"].item()) == len(oc)
            assert np.array_equal(lv["coors"][: len(oc)].cpu().numpy(), oc)
            ref = S.neighbor_table(cur, shape, oc, p["ks"], p["st"], p["pd"])
            assert np.array_equal(p["nbr"][: len(oc)].cpu().numpy(), ref)
            cur, shape, lvl = oc, oshape, lvl + 1
    assert shape == (2, 200, 176)


def _weights(seed=3):
    from sessd_b200 import weights
    sd = weights.random_detector_state(seed)
    return weights.split_detector_state(sd)


@pytest.mark.parametrize("use_tc,split,rows,kw", [(False, None, 0, {}), (True, "fp16", 16, dict(sparse_tc="cg", keep_f32=True)), (True, "fp16", 16, {})],
                         ids=["simt", "rows16+pair-gather+f32rows", "rows16+pair-gather(default)"])
def test_spmiddle_features_match_fp64_oracle(use_tc, split, rows, kw):
    from oracle import spconv_ref as S
    from sessd_b200 import synth
    from sessd_b200.runners import SpMiddleRunner
    v, coors, num = _voxels(synth.ring_cloud(5, 8000))
    n = len(coors)
    feat = (v.sum(1) / num[:, None]).astype(np.float32)
    layers, _, _ = _weights()
    params = [dict(weight=l["weight"].numpy(), gamma=l["gamma"].numpy(), beta=l["beta"].numpy(), mean=l["mean"].numpy(),
                   var=l["var"].numpy()) for l in layers]
    trace = []
    ref = S.spmiddle_forward(feat, coors, 1, (1408, 1600, 40), params, np.float64, trace)   # [1,128,200,176]
    r = SpMiddleRunner(1, n, device="cuda", use_tc=use_tc, split=split, rows_max_cin=rows, **kw)
    assert [p["impl"] for p in r.plan].count("rows") == {0: 0, 16: 3, 32: 5}[rows]
    if use_tc and split == "fp16" and rows == 16:
        assert [p["impl"] for p in r.plan].count(kw.get("sparse_tc", "cg")) == 11
    r.load_weights(layers)
    dense = r.forward(torch.from_numpy(feat).cuda(), torch.from_numpy(coors).cuda(), torch.tensor([n], dtype=torch.int32, device="cuda"))
    torch.cuda.synchronize()
    for li, t in enumerate(trace):
        got = r.layer_output(li)[: len(t["coors"])].cpu().numpy().astype(np.float64)
        scale = np.abs(t["feat"]).max() + 1e-30
        assert np.abs(got - t["feat"]).max() / scale < 1e-5, "layer %d" % li
    got = dense.permute(0, 3, 1, 2).cpu().numpy().astype(np.float64)     # NHWC storage -> logical NCHW
    assert got.shape == ref.shape
    assert np.abs(got - ref).max() / np.abs(ref).max() < 1e-5
    assert ((got != 0) == (ref != 0)).all()


def _full_size_runner(n_frames=4, pts=200000, **kw):
    """BASELINE config #5-style clouds (uniform 200 k points per frame) through the voxeliser + SpMiddleRunner on the device."""
    from sessd_b200 import ops, synth
    from sessd_b200.runners import SpMiddleRunner
    clouds = [synth.uniform_cloud(500 + f, pts) for f in range(n_frames)]
    cfg = ops.make_voxel_cfg(synth.VOXEL_SIZE, synth.PC_RANGE, 5, 200000)
    total = sum(c.shape[0] for c in clouds)
    vox = ops.VoxelBuffers(cfg, n_frames, total, "cuda", with_mean=True)
    off = np.zeros(n_frames + 1, np.int32)
    off[1:] = np.cumsum([c.shape[0] for c in clouds])
    ops.voxelize(torch.from_numpy(np.concatenate(clouds, 0)).cuda(), torch.from_numpy(off).cuda(), vox)
    r = SpMiddleRunner(n_frames, n_frames * 200000, device="cuda", growth=(1.0, 8.0, 8.0, 8.0, 8.0), **kw)
    layers, _, _ = _weights()
    r.load_weights(layers)
    return r, vox, n_frames


def test_full_size_rulebook_symmetry_and_conv_properties():
    """Size-independent properties at the stress shape (4 frames x 200 k points, ~0.8 M voxels, up to 3 M active sites):
    * SubM rulebook symmetry: nbr[o][k] = i  <=>  nbr[i][26-k] = o, centre offset = identity, rows in range;
    * strided levels: output coordinates strictly ascending in linear index (canonical order), every output has >= 1 input;
    * the tensor-core and the SIMT sparse-conv implementations agree layer by layer (<= 1e-5 of the layer maximum) and are run-to-run deterministic (bitwise);
    * dense(): the one-pass gather equals memset + scatter bitwise."""
    from sessd_b200 import ops
    from sessd_b200.runners import SpMiddleRunner
    r, vox, B = _full_size_runner()
    n0 = vox.num_voxels[B:B + 1]
    d1 = r.forward(vox.mean, vox.coors, n0).clone()
    torch.cuda.synchronize()
    assert int(r.status.item()) == 0
    feats1 = [r.layer_output(li).clone() for li in range(len(r.plan))]
    # --- rulebooks
    seen = set()
    for p in r.plan:
        n = int((n0 if p["lout"] == 0 else r.levels[p["lout"]]["n"]).item())
        nbr = p["nbr"][:n].long()
        if p["kind"] == "subm":
            if p["key"] in seen:
                continue
            seen.add(p["key"])
            ar = torch.arange(n, device="cuda")
            assert torch.equal(nbr[:, 13], ar)
            assert int(nbr.max()) < n and int(nbr.min()) >= -1
            for k in (0, 5, 12):
                o = torch.nonzero(nbr[:, k] >= 0).squeeze(1)
                i = nbr[o, k]
                assert torch.equal(nbr[i, 26 - k], o), (p["key"], k)
        else:
            lv = r.levels[p["lout"]]
            c = lv["coors"][:n].long()
            d, h, w = lv["shape"]
            lin = ((c[:, 0] * d + c[:, 1]) * h + c[:, 2]) * w + c[:, 3]
            assert bool((lin[1:] > lin[:-1]).all())
            assert bool((nbr >= 0).any(dim=1).all())
    # --- determinism + agreement between implementations
    d2 = r.forward(vox.mean, vox.coors, n0)
    torch.cuda.synchronize()
    assert torch.equal(d1, d2)
    for li, a in enumerate(feats1):
        assert torch.equal(a, r.layer_output(li))
    counts = [int((n0 if p["lout"] == 0 else r.levels[p["lout"]]["n"]).item()) for p in r.plan]
    for kw in (dict(use_tc=False),):
        q = SpMiddleRunner(B, B * 200000, device="cuda", growth=(1.0, 8.0, 8.0, 8.0, 8.0), **kw)
        q.load_weights(_weights()[0])
        dq = q.forward(vox.mean, vox.coors, n0)
        torch.cuda.synchronize()
        for li, (a, b) in enumerate(zip(feats1, q.feats)):
            n = counts[li]
            scale = float(a[:n].abs().max()) + 1e-30
            assert float((a[:n] - b[:n]).abs().max()) / scale < 1e-5, (kw, li)
        assert float((dq - d1).abs().max()) / float(d1.abs().max()) < 1e-5
        # the occupancy pattern is the same; only ReLU outputs within rounding of zero may flip between implementations
        flips = (dq != 0) != (d1 != 0)
        assert float(torch.maximum(dq, d1)[flips].max() if bool(flips.any()) else 0.0) < 1e-5 * float(d1.abs().max())
        del q
    # --- dense(): gather == memset + scatter
    last = r.levels[-1]
    ref = ops.sparse_to_dense(r.feats[-1], last["coors"], last["n"], last["cap"], last["grid"], torch.empty_like(d1))
    torch.cuda.synchronize()
    assert torch.equal(ref, d1)


def test_h2_sparse_conv_power_of_two_scaling_is_exact():
    """Linearity property of the fp16-split tensor-core layer: the activation scale is an exact power of two taken from the tensor's
    abs-max, so conv(4 x) == 4 conv(x) BITWISE (shift = 0, ReLU on), at 300 k rows with a real SubM rulebook."""
    from sessd_b200 import ops
    r, vox, B = _full_size_runner(n_frames=2, pts=150000)
    n0 = vox.num_voxels[B:B + 1]
    r.forward(vox.mean, vox.coors, n0)
    torch.cuda.synchronize()
    p = r.plan[7]                                   # a 64 -> 64 SubM layer on level 2
    lv = r.levels[p["lout"]]
    n, cap = lv["n"], lv["cap"]
    x = r.layer_output(6).clone()
    w = torch.randn((27, 64, 64), device="cuda") * 0.05
    tiles, inv = ops.pack_weight_sp_h2(w, 64)
    sc = (torch.rand(64, device="cuda") + 0.5) * inv
    nn = int(n.item())
    assert nn > 100000
    # the pair-gather kernel (default): the property holds with the bound-derived scale, for fp32 rows and plane outputs
    gain = ops.conv_gain(w, sc / inv)
    tl = ops.rulebook_tile_lists(p["nbr"], n, cap, ops.alloc_tile_lists(cap, 27, "cuda"))
    cg = []
    for mul in (1.0, 4.0):
        xx = (x * mul).contiguous()
        info = torch.zeros(2, device="cuda")
        ops.absmax_rows(xx, n, cap, info[0:1])
        planes = ops.alloc_planes(cap, 64, "cuda")
        info[1] = 2.0 ** (14 - np.floor(np.log2(float(info[0]))))          # any exact power of two that keeps the planes in range
        s = float(info[1])
        hi = (xx * s).half()
        planes[:cap, :64] = hi
        planes[:cap, 64:] = (xx * s - hi.float()).half()
        out = torch.zeros((cap, 64), device="cuda")
        oplanes = ops.alloc_planes(cap, 64, "cuda")
        oinfo = torch.zeros(2, device="cuda")
        ops.spconv_forward_cg(planes, info, tl, n, cap, tiles, sc.contiguous(), None, True, gain, 0.0, out, oplanes, oinfo)
        torch.cuda.synchronize()
        back = ops.sparse_planes_to_float(oplanes[:-1], oinfo, 64)
        assert float((back[:nn] - out[:nn]).abs().max()) <= 3e-7 * float(out[:nn].abs().max())
        assert float(oinfo[0]) == float(out[:nn].abs().max())
        cg.append((out, float(oinfo[0])))
    assert torch.equal(cg[0][0][:nn] * 4.0, cg[1][0][:nn])
    assert cg[0][1] * 4.0 == cg[1][1]


# ---------------------------------------------------------------------------------------------------- BASELINE shapes (SURVEY 8d)
def _frame_through_runner(cloud, max_voxels=20000, growth=None):
    from oracle import cpu as ocpu
    from sessd_b200 import synth
    from sessd_b200.runners import SpMiddleRunner
    v, c, num = ocpu.points_to_voxel(cloud, synth.VOXEL_SIZE, synth.PC_RANGE, 5, max_voxels)
    coors = np.concatenate([np.zeros((len(c), 1), np.int32), c], 1).astype(np.int32)
    n = len(coors)
    feat = (v.sum(1) / num[:, None]).astype(np.float32)
    r = SpMiddleRunner(1, n, device="cuda", growth=growth)
    layers, _, _ = _weights()
    r.load_weights(layers)
    dense = r.forward(torch.from_numpy(feat).cuda(), torch.from_numpy(coors).cuda(), torch.tensor([n], dtype=torch.int32, device="cuda"))
    torch.cuda.synchronize()
    assert int(r.status.item()) == 0
    return r, feat, coors, layers, dense


def _check_rulebooks(r, coors):
    """all 8 rulebooks (nbr tables) and the 4 strided coordinate lists of the frame vs the oracle, bit-exact"""
    from oracle import spconv_ref as S
    cur, shape, lvl, seen = coors, (41, 1600, 1408), 0, set()
    sites = [len(coors)]
    for p in r.plan:
        if p["kind"] == "subm":
            if p["key"] in seen:
                continue
            seen.add(p["key"])
            ref = S.neighbor_table(cur, shape, cur, p["ks"], (1, 1, 1), (1, 1, 1))
            assert np.array_equal(p["nbr"][: len(cur)].cpu().numpy(), ref), p["key"]
        else:
            oc, oshape = S.strided_out_coors(cur, shape, p["ks"], p["st"], p["pd"])
            lv = r.levels[lvl + 1]
            assert int(lv["n"].item()) == len(oc)
            assert np.array_equal(lv["coors"][: len(oc)].cpu().numpy(), oc)
            ref = S.neighbor_table(cur, shape, oc, p["ks"], p["st"], p["pd"])
            assert np.array_equal(p["nbr"][: len(oc)].cpu().numpy(), ref)
            cur, shape, lvl = oc, oshape, lvl + 1
            sites.append(len(oc))
    assert shape == (2, 200, 176)
    return sites


@pytest.mark.parametrize("kind", ["ring", "uniform"])
def test_rulebooks_bit_exact_on_full_20k_frames(kind):
    """BASELINE config #2 inputs, one full frame each: ring-20k and uniform-20k (SURVEY 8(d): 20 k -> 68 k -> 103 k -> 86 k -> 52 k sites)."""
    from sessd_b200 import synth
    cloud = synth.ring_cloud(0, 20000) if kind == "ring" else synth.uniform_cloud(0, 20000)
    r, _feat, coors, _layers, _dense = _frame_through_runner(cloud)
    sites = _check_rulebooks(r, coors)
    if kind == "uniform":
        assert sites == [19998, 67955, 103374, 85774, 52169]          # SURVEY.md 8(d) [probe] counts of seed 0


def test_rulebooks_bit_exact_on_a_200k_point_frame():
    """BASELINE config #5 input (uniform-200k, max_voxels 200000), one frame: every rulebook and coordinate list vs the oracle."""
    from sessd_b200 import synth
    r, _feat, coors, _layers, _dense = _frame_through_runner(synth.uniform_cloud(1000, 200000), 200000, growth=(1.0, 8.0, 8.0, 8.0, 8.0))
    sites = _check_rulebooks(r, coors)
    assert sites[0] > 190000 and max(sites) > 600000


def test_features_uniform20k_match_fp64_oracle():
    """Per-layer features of the DEFAULT kernels on the uniform-20k frame (SURVEY 8(d) primary input) vs the fp64 oracle:
    <= 1e-5 of the layer maximum (north_star bar: 1e-4 relative)."""
    from oracle import spconv_ref as S
    from sessd_b200 import synth
    r, feat, coors, layers, dense = _frame_through_runner(synth.uniform_cloud(0, 20000))
    params = [dict(weight=l["weight"].numpy(), gamma=l["gamma"].numpy(), beta=l["beta"].numpy(), mean=l["mean"].numpy(),
                   var=l["var"].numpy()) for l in layers]
    trace = []
    ref = S.spmiddle_forward(feat, coors, 1, (1408, 1600, 40), params, np.float64, trace)
    for li, t in enumerate(trace):
        got = r.layer_output(li)[: len(t["coors"])].cpu().numpy().astype(np.float64)
        scale = np.abs(t["feat"]).max() + 1e-30
        assert np.abs(got - t["feat"]).max() / scale < 1e-5, "layer %d" % li
    got = dense.permute(0, 3, 1, 2).cpu().numpy().astype(np.float64)
    assert np.abs(got - ref).max() / np.abs(ref).max() < 1e-5


def test_tile_lists_regroup_the_neighbour_table_exactly():
    """sessd_rulebook_tile_lists (the rulebook format of the pair-gather conv) vs a numpy regrouping of the same nbr table: counts, row masks
    and the (input row << 7 | tile row) entries per offset in ascending tile row -- bit-exact, SubM (kvol 27) and the (3,1,1) layer (kvol 3)."""
    from sessd_b200 import ops, synth
    r, _feat, coors, _layers, _dense = _frame_through_runner(synth.ring_cloud(3, 20000))
    for p in (r.plan[3], r.plan[6], r.plan[13]):
        n = int((r.levels[p["lout"]]["n"]).item())
        kvol = p["nbr"].shape[1]
        cap = p["nbr"].shape[0]
        tl = ops.rulebook_tile_lists(p["nbr"], r.levels[p["lout"]]["n"], cap, ops.alloc_tile_lists(cap, kvol, "cuda"))
        torch.cuda.synchronize()
        nbr = p["nbr"][:n].cpu().numpy()
        rec = tl.cpu().numpy().view(np.uint32)
        stride = rec.shape[1]
        assert stride == 160 + 128 * kvol
        for t in range(-(-n // 128)):
            rows = nbr[t * 128:(t + 1) * 128]
            pos = 160
            for k in range(kvol):
                valid = np.nonzero(rows[:, k] >= 0)[0]
                assert rec[t, k] == len(valid), (t, k)
                mask = np.zeros(4, np.uint32)
                for rr in valid:
                    mask[rr >> 5] |= np.uint32(1) << np.uint32(rr & 31)
                assert np.array_equal(rec[t, 32 + 4 * k:36 + 4 * k], mask), (t, k)
                want = (rows[valid, k].astype(np.uint32) << np.uint32(7)) | valid.astype(np.uint32)
                assert np.array_equal(rec[t, pos:pos + len(valid)], want), (t, k)
                pos += len(valid)
            assert not rec[t, kvol:32].any()
