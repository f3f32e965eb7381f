"""The training-workspace reader and the stage comparators of tests/train_tape.py, without a GPU.

A synthetic "device" is built in numpy from the oracle: the fp16 forward tape with its sign bits, the compositing
backward, dd and the dgrad chain with per-level power-of-two scales, and the gradients contracted from those stored
values - what a correct training step leaves behind.  The comparators must accept it, and each must reject it once
one defect of the kind it exists for is injected.  So the bars are not so wide that they pass everything."""
import numpy as np
import pytest

from oracle import nerf_oracle as orc
from oracle import nerf_oracle_grad as og
from tests import train_tape as tt

F32, F64 = np.float32, np.float64


# ------------------------------------------------------------------------------------------ layouts
def test_untile_follows_layout_h():
    """Element (row r, column k) of a tiled (n, C) array: block (r / 64, k / 64) at ((r / 64) (C / 64) + k / 64) 8 KiB,
    inside it at (r % 64) 128 + (((k % 64) >> 3) ^ (r & 7)) 16 + (k & 7) 2 (csrc/layout.h)."""
    rs = np.random.RandomState(0)
    n, C = 256, 128
    x = rs.randn(n, C).astype(np.float16)
    raw = np.zeros(n * C * 2, np.uint8)
    for r in range(n):
        for k in range(C):
            kk = k % 64
            off = ((r // 64) * (C // 64) + k // 64) * 8192 + (r % 64) * 128 + (((kk >> 3) ^ (r & 7)) << 4) + (kk & 7) * 2
            raw[off:off + 2] = x[r:r + 1, k].view(np.uint8)
    np.testing.assert_array_equal(tt.untile(raw, n, C), x)
    np.testing.assert_array_equal(tt.tile(x), raw)
    np.testing.assert_array_equal(tt.untile(raw, n, C, np.array([3, 1])), x[np.r_[192:256, 64:128]])


def test_decode_masks_follows_epi_hidden():
    """csrc/mlp_engine.cuh epi_hidden: bit 2 (j & 15) + e of word j >> 4 of entry (row, q) is the sign of column
    8 j + 2 q + e.  One bit at a time."""
    for j, q, e in [(0, 0, 0), (0, 0, 1), (1, 0, 0), (0, 1, 0), (0, 3, 1), (15, 2, 1), (16, 0, 0), (17, 1, 1), (31, 3, 1)]:
        m = np.zeros((1, 4, 2), np.uint32)
        m[0, q, j >> 4] = np.uint32(1) << np.uint32(2 * (j & 15) + e)
        neg = tt.decode_masks(m)
        assert np.flatnonzero(neg[0]).tolist() == [8 * j + 2 * q + e], (j, q, e)
    rs = np.random.RandomState(1)
    neg = rs.rand(40, 256) < 0.5
    np.testing.assert_array_equal(tt.decode_masks(tt.encode_masks(neg)), neg)


def test_layout_matches_workspace_size_order():
    """The per-pass buffers follow each other in make_train_layout's order, 1 KiB aligned, fine after coarse."""
    L = tt.layout(33, 32, 32)
    assert [P["S"] for P in L] == [32, 64]
    assert L[0]["n_pad"] == 1152 and L[1]["n_pad"] == 2176
    keys = ["enc", "act", "mask", "d", "sigma", "rgb", "z", "dsigma", "dprergb", "dd", "dpre"]
    offs = [P[k] for P in L for k in keys]
    assert offs == sorted(offs) and all(o % 1024 == 0 for o in offs)
    assert L[0]["act"] - L[0]["enc"] == 1152 * 128 and L[1]["enc"] == L[0]["dpre"] + 1152 * 512 * 8


def test_column_sums_round_like_the_fp16_pre_sums():
    """8 rows (h 32 + 4 i + p) are added in fp16 first: 2048 + 1 + 1 stays 2048 there (ties to even), the rest
    of the chunk is exact."""
    a = np.zeros((64, 2), np.float16)
    a[[0, 4, 8], 0] = [2048, 1, 1]       # one 8-row group: 2048
    a[[0, 1, 2], 1] = [2048, 1, 1]       # three groups: 2050
    np.testing.assert_array_equal(tt.column_sums(a), [2048.0, 2050.0])


def test_pow2_ratio_rejects_a_non_power_of_two():
    x = np.linspace(1, 2, 100)
    assert tt.pow2_ratio(x * 8, x) == 8.0
    with pytest.raises(AssertionError):
        tt.pow2_ratio(x * 3, x)


# ------------------------------------------------------------------------------------------ synthetic device
def _f16(x):
    return np.asarray(x, F32).astype(np.float16)


def synthetic(n_rays=16, S=64):
    """What a correct training step leaves for one coarse-only pass, emulated in numpy (fp16 storage, fp32 math)."""
    w = orc.make_weights(11)
    net = tt.Net(w)
    rays = orc.make_rays(n_rays, 5)
    rs = np.random.RandomState(2)
    z = orc.coarse_depths(rays, S, False, 1.0, rs.rand(n_rays, S).astype(F32))
    o, d = rays[:, :3], rays[:, 3:6]
    dir_emb = orc.embed(d, 4)
    xyz = (o[:, None] + d[:, None] * z[:, :, None]).astype(F32).reshape(-1, 3)
    enc = np.zeros((len(xyz), 64), np.float16)
    enc[:, :63] = _f16(orc.embed(xyz, 10))
    x = enc[:, :63].astype(F64)
    hs, negs, prev = [], [], x
    for l in range(1, 9):
        inp = np.concatenate([x, prev], 1) if l == 5 else prev
        pre = (inp @ net.W[l].T + net.b[l]).astype(F32)
        negs.append(pre < 0)
        hs.append(_f16(np.maximum(pre, 0)))
        prev = hs[-1].astype(F64)
    rows = np.arange(len(xyz)) // S
    pre8 = (prev @ net.Wp.T + net.bp + dir_emb[rows] @ net.Wdir.T).astype(F32)
    dv = _f16(np.maximum(pre8, 0))
    sigma = (net.bsig + np.maximum(hs[7].astype(F64), 0) @ net.wsig).astype(F32)
    rgb = (1 / (1 + np.exp(-(dv.astype(F64) @ net.Wrgb.T + net.brgb)))).astype(F32)
    _, rgb_out, _, _ = orc.volume_render(sigma.reshape(n_rays, S), rgb.reshape(n_rays, S, 3), z, d, None, 0.0, True)
    target = rs.uniform(0, 1, (n_rays, 3)).astype(F32)
    g_rgb = (2.0 * (rgb_out - target) / (3 * n_rays)).astype(F32)
    dsig, drgb = og.volume_render_backward(sigma.reshape(n_rays, S), rgb.reshape(n_rays, S, 3), z, d, None, 0.0, True,
                                           g_rgb)
    dsig = dsig.reshape(-1)
    dprergb = (drgb.reshape(-1, 3).astype(F64) * rgb * (1 - rgb.astype(F64))).astype(F32)
    ref0 = (dprergb.astype(F64) @ net.Wrgb) * (dv > 0)
    bound = max(np.abs(dprergb).max() * np.abs(net.Wrgb).sum(0).max(), np.abs(dsig).max() * np.abs(net.wsig).max())
    scales = [2.0 ** np.floor(np.log2(64 / bound))]
    dd = _f16(ref0 * scales[0])
    a = dd.astype(F64) @ net.Wp + (dsig.astype(F64) * scales[0])[:, None] * net.wsig[None, :]
    dpre = [None] * 8
    for v in range(1, 9):
        l = 9 - v
        val = a * ~negs[l - 1]
        s = 2.0 ** np.floor(np.log2(64 / (np.abs(val).max() / scales[-1])))
        dpre[l - 1] = _f16(val * (s / scales[-1]))
        scales.append(s)
        if l > 1:
            a = dpre[l - 1].astype(F64) @ net.Wchain(l)
    arrays = dict(z=z, enc=enc, h=hs, neg=negs, d=dv, sigma=sigma, rgb=rgb, dsigma=dsig, dprergb=dprergb, dd=dd,
                  dpre=dpre)
    return dict(net=net, rays=rays, dir_emb=dir_emb, arrays=arrays, scales=scales, g_rgb=g_rgb, S=S)


def device_grads(syn):
    """The gradients a correct wgrad / reduction / unfold produces from the stored arrays (fp32 results)."""
    tape = tt.ArrayTape(syn["S"], syn["arrays"])
    return {k: v.astype(F32) for k, v in tt.reference_grads(tape, syn["net"], syn["scales"], syn["dir_emb"]).items()}


def all_failures(syn, grads):
    tape = tt.ArrayTape(syn["S"], syn["arrays"])
    fwd = tt.check_forward(tape, syn["net"], syn["dir_emb"])
    masks = tt.check_masks(tape)
    comp = tt.check_composite(tape, syn["rays"], syn["g_rgb"], None, None, None, 0.0, True)
    chain = tt.check_chain(tape, syn["net"])
    ref = tt.reference_grads(tape, syn["net"], chain["scales"], syn["dir_emb"])
    return tt.failures(fwd, masks, chain, comp, tt.check_grads(grads, ref))


@pytest.fixture(scope="module")
def syn():
    return synthetic()


def _fresh(syn):
    a = syn["arrays"]
    arrays = dict(a, h=list(a["h"]), neg=[x.copy() for x in a["neg"]], dpre=[x.copy() for x in a["dpre"]])
    return dict(syn, arrays=arrays)


def workspace_bytes(syn):
    """The synthetic pass written into a workspace byte image at make_train_layout's offsets (n_pad rows)."""
    S, a = syn["S"], syn["arrays"]
    n_rays = len(syn["rays"])
    P = tt.layout(n_rays, S, 0)[0]
    n, npad = P["n"], P["n_pad"]
    raw = np.zeros(P["dpre"] + npad * 512 * 8 + 1024, np.uint8)

    def put(off, arr):
        b = np.ascontiguousarray(arr).view(np.uint8).reshape(-1)
        raw[off:off + b.size] = b

    def pad(x):
        out = np.zeros((npad,) + x.shape[1:], x.dtype)
        out[:n] = x
        return out
    put(P["enc"], tt.tile(pad(a["enc"])))
    for l in range(8):
        put(P["act"] + l * npad * 512, tt.tile(pad(a["h"][l])))
        put(P["dpre"] + l * npad * 512, tt.tile(pad(a["dpre"][l])))
        put(P["mask"] + l * npad * 32, tt.encode_masks(pad(a["neg"][l])))
    put(P["d"], tt.tile(pad(a["d"])))
    put(P["dd"], tt.tile(pad(a["dd"])))
    for k in ("sigma", "rgb", "dsigma", "dprergb"):
        put(P[k], pad(a[k].astype(F32)))
    put(P["z"], a["z"].astype(F32))
    return raw, P


def test_workspace_reader_round_trip(syn):
    """WorkspaceTape reads back, from the byte image, exactly the arrays written at the mirrored offsets - for all
    rows and for a tile subset."""
    raw, P = workspace_bytes(syn)
    a = syn["arrays"]
    for tiles in (None, np.array([5, 1])):
        tape = tt.WorkspaceTape(raw, P, tiles)
        r = tape.rows
        np.testing.assert_array_equal(tape.z(), a["z"])
        for k in ("sigma", "rgb", "dsigma", "dprergb", "enc", "d", "dd"):
            np.testing.assert_array_equal(getattr(tape, k)(), a[k][r], err_msg=k)
        for l in range(1, 9):
            np.testing.assert_array_equal(tape.h(l), a["h"][l - 1][r])
            np.testing.assert_array_equal(tape.dpre(l), a["dpre"][l - 1][r])
            np.testing.assert_array_equal(tape.neg(l), a["neg"][l - 1][r])
    assert tape.saturated() == 0
    full = tt.WorkspaceTape(raw, P)
    assert tt.failures(chain=tt.check_chain(full, syn["net"])) == []


def test_reference_grads_do_not_depend_on_the_parts():
    """reference_grads of a workspace summed one tile at a time equals the sum over the whole array tape to float64
    rounding: 96-sample rays straddle the parts, and the last tile, a part of its own, is half padding."""
    syn = synthetic(5, 96)
    raw, P = workspace_bytes(syn)
    whole = tt.reference_grads(tt.ArrayTape(syn["S"], syn["arrays"]), syn["net"], syn["scales"], syn["dir_emb"])
    tape = tt.WorkspaceTape(raw, P)
    assert len(tape.parts(1)) == P["n_pad"] // 128 > 2
    for k, v in tt.reference_grads(tape, syn["net"], syn["scales"], syn["dir_emb"], tiles_per_part=1).items():
        np.testing.assert_allclose(v, whole[k], rtol=1e-12, atol=1e-12 * np.abs(whole[k]).max(), err_msg=k)


def test_correct_device_passes(syn):
    assert all_failures(syn, device_grads(syn)) == []
    chain = tt.check_chain(tt.ArrayTape(syn["S"], syn["arrays"]), syn["net"])
    assert chain["scales"] == syn["scales"]


def test_dropped_wgrad_chunk_is_caught(syn):
    """One 64-sample chunk missing from sum_s dpre_3^T h_2."""
    g = device_grads(syn)
    a = syn["arrays"]
    A = a["dpre"][2][128:192].astype(F64) / syn["scales"][6]
    g["xyz_encoding_3.0.weight"] = (g["xyz_encoding_3.0.weight"] - A.T @ a["h"][1][128:192].astype(F64)).astype(F32)
    bad = all_failures(syn, g)
    assert bad and all("xyz_encoding_3.0.weight" in b for b in bad), bad


def test_swapped_mask_columns_are_caught(syn):
    """Sign bits decoded for the wrong column: two columns of one 16-column group swapped in layer 6's mask."""
    s = _fresh(syn)
    neg = s["arrays"]["neg"][5]
    neg[:, [18, 21]] = neg[:, [21, 18]]
    bad = all_failures(s, device_grads(syn))
    assert any(b.startswith("masks") for b in bad), bad


def test_missing_direction_slice_is_caught(syn):
    """One dir_grad_kernel slice that never writes its partial: the rays of slice 3 drop out of gW_dir[:, 256:]."""
    g = device_grads(syn)
    tape = tt.ArrayTape(syn["S"], syn["arrays"])
    ref0, _ = tt.dd_reference(tape, syn["net"])
    n_rays = len(syn["rays"])
    per = -(-n_rays // tt.DIR_SLICES)
    r = np.arange(3 * per, min(4 * per, n_rays))
    assert len(r)
    raysum = ref0.reshape(n_rays, syn["S"], 128).sum(1)
    g["dir_encoding.0.weight"] = g["dir_encoding.0.weight"].copy()
    g["dir_encoding.0.weight"][:, 256:] -= (raysum[r].T @ syn["dir_emb"][r].astype(F64)).astype(F32)
    bad = all_failures(syn, g)
    assert bad and all("dir_encoding.0.weight" in b for b in bad), bad


def test_level_stored_at_twice_its_scale_is_caught(syn):
    """dpre_4 stored at twice the scale the reduction un-scales it with: the chain stays self-consistent, the
    gradient of layer 4 doubles."""
    s = _fresh(syn)
    s["arrays"]["dpre"][3] = _f16(s["arrays"]["dpre"][3].astype(F64) * 2)
    bad = all_failures(s, device_grads(s))
    assert any("xyz_encoding_4.0" in b for b in bad), bad


def test_saturated_element_is_caught(syn):
    s = _fresh(syn)
    s["arrays"]["dpre"][6][100, 7] = np.float16(65504.0)
    bad = all_failures(s, device_grads(s))
    assert any("saturated" in b for b in bad), bad
