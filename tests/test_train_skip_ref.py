"""The float64 restatement of the training step with empty samples skipped (tests/train_skip_ref.py): its closed-form
sparse compositing backward equals torch autograd in float64, skipped samples carry neither weight nor gradient, and
each comparison the GPU tests make with it rejects a planted defect."""
import numpy as np
import pytest
import torch

from tests import train_skip_ref as tr


def _case(R=6, S=64, seed=0, white_back=True, noise_std=1.0):
    rng = np.random.default_rng(seed)
    near, far = 2.0, 6.0
    z = np.sort(rng.uniform(near, far, (R, S)), 1)
    sigma = rng.normal(2.0, 3.0, (R, S))
    rgb = rng.uniform(0.05, 0.95, (R, S, 3))
    ev = rng.random((R, S)) < 0.4
    ev[0] = True                     # a ray with nothing skipped
    ev[1] = False                    # a ray with every sample skipped
    dirs = rng.normal(size=(R, 3))
    noise = rng.normal(size=(R, S))
    target = rng.uniform(0, 1, (R, 3))
    return dict(z=z, sigma=sigma, rgb=rgb, ev=ev, dirs=dirs, noise=noise, noise_std=noise_std, white_back=white_back,
                target=target)


def _autograd(c):
    z = torch.tensor(c["z"])
    s = torch.tensor(c["sigma"], requires_grad=True)
    pre = torch.logit(torch.tensor(c["rgb"])).requires_grad_(True)
    ev = torch.tensor(c["ev"])
    sig = torch.where(ev, s + torch.tensor(c["noise"]) * c["noise_std"], torch.zeros_like(s))
    rgb = torch.where(ev[..., None], torch.sigmoid(pre), torch.zeros_like(pre))
    out, _, _ = tr.composite_torch(z, sig, rgb, torch.tensor(c["dirs"]), c["white_back"])
    loss = ((out - torch.tensor(c["target"])) ** 2).mean()
    loss.backward()
    return out.detach().numpy(), s.grad.numpy(), pre.grad.numpy()


def _closed(c, out):
    return tr.backward(c["z"], c["sigma"], c["rgb"], c["ev"], c["dirs"], c["noise"], c["noise_std"], c["white_back"],
                       out, c["target"], c["z"].shape[0])


@pytest.mark.parametrize("white_back,noise_std", [(True, 1.0), (False, 0.0), (False, 1.0)])
def test_closed_form_backward_is_autograd(white_back, noise_std):
    c = _case(white_back=white_back, noise_std=noise_std, seed=int(white_back) + 2 * int(noise_std))
    out, ds_ref, dp_ref = _autograd(c)
    ds, dp = _closed(c, out)
    assert np.allclose(ds, ds_ref, rtol=1e-9, atol=1e-15) and np.allclose(dp, dp_ref, rtol=1e-9, atol=1e-15)
    assert not ds[~c["ev"]].any() and not dp[~c["ev"]].any()
    assert not ds[1].any() and not dp[1].any()


def test_forward_matches_autograd_and_skips():
    c = _case()
    smp = np.concatenate([c["rgb"], c["sigma"][..., None]], -1) * c["ev"][..., None]
    rays = np.concatenate([np.zeros((6, 3)), c["dirs"], np.zeros((6, 2))], 1)
    ref = tr.forward(c["z"], smp, c["ev"], rays, c["noise"], c["noise_std"], c["white_back"])
    out, _, _ = _autograd(c)
    assert np.allclose(ref["rgb"], out, atol=1e-12)
    assert not ref["weights"][~c["ev"]].any()
    assert np.allclose(ref["rgb"][1], 1.0) and ref["opacity"][1] == 0.0         # the vacuum value


def test_planted_defects_are_rejected():
    """The comparisons the GPU tests make (assert_close on the forward, backward_errors at BWD_BAR on the per-row
    gradients) reject a kernel with one defect of the kinds they exist for, emulated here in float32."""
    c = _case()
    ev = c["ev"]
    smp = np.concatenate([c["rgb"], c["sigma"][..., None]], -1) * ev[..., None]
    rays = np.concatenate([np.zeros((6, 3)), c["dirs"], np.zeros((6, 2))], 1)
    ref = tr.forward(c["z"], smp, ev, rays, c["noise"], c["noise_std"], c["white_back"])
    dev = {k: ref[k].astype(np.float32) for k in ("rgb", "depth", "opacity")}
    tr.assert_close(ref, dev, ref["weights"].astype(np.float32), ref_weights=True)
    # forward defect: noise added to skipped samples (they composite as evaluated samples of sigma 0 + noise)
    noisy = tr.forward(c["z"], smp, np.ones_like(ev), rays, c["noise"], c["noise_std"], c["white_back"])
    with pytest.raises(AssertionError):
        tr.assert_close(ref, {k: noisy[k].astype(np.float32) for k in ("rgb", "depth", "opacity")},
                        noisy["weights"].astype(np.float32), ref_weights=True)
    out = ref["rgb"]
    ds_ref, dp_ref = _closed(c, out)
    good = tr.backward_errors(ds_ref[ev].astype(np.float32), dp_ref[ev].astype(np.float32), ev, ds_ref, dp_ref)
    assert max(good) <= tr.BWD_BAR
    defects = {
        "noise dropped": dict(noise_std=0.0),
        "white_back ignored": dict(white_back=not c["white_back"]),
        "skipped samples given sigma = noise": dict(ev=np.ones_like(ev)),
    }
    for name, kw in defects.items():
        d = dict(c, **kw)
        bad_ds, bad_dp = tr.backward(d["z"], d["sigma"], d["rgb"], d["ev"], d["dirs"], d["noise"], d["noise_std"],
                                     d["white_back"], out, d["target"], d["z"].shape[0])
        errs = tr.backward_errors(bad_ds[ev].astype(np.float32), bad_dp[ev].astype(np.float32), ev, ds_ref, dp_ref)
        assert max(errs) > tr.BWD_BAR, (name, errs)
    # the ReLU mask dropped from d sigma
    s = c["sigma"] + c["noise"] * c["noise_std"]
    z = c["z"]
    delta = np.concatenate([z[:, 1:] - z[:, :-1], np.full((6, 1), 1e10)], 1) * np.linalg.norm(c["dirs"], axis=1)[:, None]
    c2 = dict(c, sigma=np.where(ev & (s <= 0), np.abs(c["sigma"]) + 5.0, c["sigma"]))
    bad_ds, _ = _closed(c2, out)
    assert (ev & (s <= 0) & (delta < 1e9)).any()
    errs = tr.backward_errors(bad_ds[ev].astype(np.float32), dp_ref[ev].astype(np.float32), ev, ds_ref, dp_ref)
    assert max(errs) > tr.BWD_BAR, errs
