"""Pins oracle/c2v_oracle.c (and the torch restatement used as the timed CPU
baseline) against outputs of the unmodified reference (tests/golden/, generated
by oracle/gen_golden.py from /root/reference/model/model.py:44-105)."""
import numpy as np
import pytest
import torch

from conftest import golden_names, load_golden
from oracle import oracle

FWD_TOL = 2e-6     # fp32 abs; the oracle is correctly-rounded per op, the rest is ATen summation order


def _forward(rec):
    ang = None
    if rec["opt"]["angular"]:
        ang = {"margin": rec["opt"]["margin"], "inverse_temp": rec["opt"]["inverse_temp"]}
    return oracle.forward(rec["params"], rec["starts"], rec["paths"], rec["ends"], rec["label"], angular=ang)


@pytest.mark.parametrize("name", golden_names())
def test_c_oracle_matches_reference_forward(name):
    rec = load_golden(name)
    out, cv, att = _forward(rec)
    scale = max(1.0, float(np.abs(rec["outputs"]).max()))
    assert np.abs(cv - rec["code_vector"]).max() <= FWD_TOL
    assert np.abs(att - rec["attention"]).max() <= FWD_TOL
    assert np.abs(out - rec["outputs"]).max() <= FWD_TOL * scale * 4
    # attention rows sum to one, also for all-pad bags (uniform 1/L, model.py:93)
    assert np.allclose(att.sum(1), 1.0, atol=1e-5)


def test_kat_matches_survey_numbers():
    """The RNG-free known-answer vector, typed in from the survey
    (independent of the .npz), incl. a mask hole and an all-pad bag."""
    rec = load_golden("kat")
    out, cv, att = _forward(rec)
    exp_out = np.array([[-0.2574855, -0.1097331, 0.6001713], [-0.3348166, -0.2768353, 0.7792008],
                        [-0.8066451, -0.0473413, 1.1113594]], np.float32)
    exp_cv = np.array([[-0.3753232, 0.1154047, 0.0589585, -0.0077963], [-0.4495981, -0.1501029, 0.2217275, 0.0306741],
                       [0.3476003, -0.6535420, -0.8808783, 0.7176104]], np.float32)
    exp_att = np.array([[0.1902112, 0.5771278, 0.2326610, 0, 0], [0.4154830, 0, 0.1474933, 0.2945327, 0.1424911],
                        [0.2, 0.2, 0.2, 0.2, 0.2]], np.float32)
    assert np.abs(out - exp_out).max() < 2e-6
    assert np.abs(cv - exp_cv).max() < 2e-6
    assert np.abs(att - exp_att).max() < 2e-6
    assert att[0, 3] == 0.0 and att[1, 1] == 0.0       # padded slots are exactly zero


@pytest.mark.parametrize("name", golden_names("grad_"))
def test_c_oracle_backward_matches_reference_autograd(name):
    rec = load_golden(name)
    out, cv, att = _forward(rec)
    loss, am, mx = oracle.loss_argmax(out, rec["label"])
    assert abs(loss - float(rec["loss"])) < 2e-6 * max(1.0, abs(loss))
    B, C = out.shape
    sm = torch.softmax(torch.from_numpy(out).double(), dim=1).numpy()
    g = sm.copy()
    g[np.arange(B), rec["label"]] -= 1.0
    g = (g / B).astype(np.float32)
    grads = oracle.backward(rec["params"], rec["starts"], rec["paths"], rec["ends"], g)
    for k, ref in rec["grads"].items():
        tol = 3e-6 * max(1.0, float(np.abs(ref).max()))
        assert np.abs(grads[k] - ref).max() <= tol, k


@pytest.mark.parametrize("name", ["tiny", "cfg2_small", "angular", "real_batch"])
def test_torch_restatement_matches_reference(name):
    """oracle.torch_forward is what bench.py times as the CPU baseline; it must be the same function."""
    rec = load_golden(name)
    p = {k: torch.from_numpy(v) for k, v in rec["params"].items()}
    ang = None
    if rec["opt"]["angular"]:
        ang = {"margin": rec["opt"]["margin"], "inverse_temp": rec["opt"]["inverse_temp"]}
    with torch.no_grad():
        out, cv, att = oracle.torch_forward(p, torch.from_numpy(rec["starts"]), torch.from_numpy(rec["paths"]),
                                            torch.from_numpy(rec["ends"]), torch.from_numpy(rec["label"]), angular=ang)
    assert np.abs(out.numpy() - rec["outputs"]).max() <= 1e-6 * max(1.0, float(np.abs(rec["outputs"]).max()))
    assert np.abs(cv.numpy() - rec["code_vector"]).max() <= 1e-6
    assert np.abs(att.numpy() - rec["attention"]).max() <= 1e-6


def _fp64_loss_and_grads(rec):
    """oracle.torch_forward in fp64 + mean NLL (main.py:251-264), autograd through every parameter and every tap"""
    p = {k: torch.from_numpy(v).double().requires_grad_() for k, v in rec["params"].items()}
    ang = None
    if rec["opt"]["angular"]:
        ang = {"margin": rec["opt"]["margin"], "inverse_temp": rec["opt"]["inverse_temp"]}
    taps = {}
    label = torch.from_numpy(rec["label"])
    out, cv, att = oracle.torch_forward(p, torch.from_numpy(rec["starts"]), torch.from_numpy(rec["paths"]),
                                        torch.from_numpy(rec["ends"]), label, angular=ang, taps=taps)
    for t in taps.values():
        t.retain_grad()
    loss = torch.nn.functional.nll_loss(torch.log_softmax(out, 1), label)
    loss.backward()
    return loss, p, taps, out


@pytest.mark.parametrize("name", golden_names("grad_") + golden_names("angular_grad"))
def test_fp64_torch_restatement_reproduces_reference_gradients(name):
    """The fp64 judge of tests/test_train_step_gpu.py (torch_forward + mean NLL, double precision) is the reference's
    autograd: same loss, same gradient of every parameter, both label heads."""
    rec = load_golden(name)
    loss, p, taps, out = _fp64_loss_and_grads(rec)
    assert abs(loss.item() - float(rec["loss"])) <= 2e-6 * max(1.0, abs(float(rec["loss"])))
    assert np.abs(out.detach().numpy() - rec["outputs"]).max() <= 2e-6 * max(1.0, float(np.abs(rec["outputs"]).max()))
    assert set(rec["grads"]) == set(p)
    for k, ref in rec["grads"].items():
        tol = 2e-6 * max(1.0, float(np.abs(ref).max()))
        assert np.abs(p[k].grad.numpy() - ref).max() <= tol, k
    # the taps are the live intermediates: d loss / d logits is softmax - one-hot over the batch
    B = out.shape[0]
    g = torch.softmax(out.detach(), 1)
    g[torch.arange(B), torch.from_numpy(rec["label"])] -= 1.0
    assert torch.allclose(taps["logits"].grad, g / B, rtol=0, atol=1e-15)
    assert taps["x"].shape == taps["ln"].shape == rec["starts"].shape + (p["input_linear.weight"].shape[0],)
    assert taps["cv"].grad.shape == out.shape[:1] + (p["input_linear.weight"].shape[0],)
    assert taps["z"].grad.shape == rec["starts"].shape
    assert ("cos" in taps) == bool(rec["opt"]["angular"])


@pytest.mark.parametrize("name", ["tiny", "cfg2_small", "grad_odd"])
def test_torch_restatement_applies_a_given_dropout_mask_like_the_c_oracle(name):
    """torch_forward(..., dropmask=) multiplies tanh's output by the mask before the scores and the weighted sum, as
    oracle.encode_forward(..., dropmask=) does (model.py:60-61 with the mask drawn by the kernels)."""
    rec = load_golden(name)
    p = rec["params"]
    B, L = rec["starts"].shape
    H = p["input_linear.weight"].shape[0]
    mask = (np.random.default_rng(5).random((B, L, H)) >= 0.25).astype(np.float32) / np.float32(0.75)
    cv, att = oracle.encode_forward(rec["starts"], rec["paths"], rec["ends"], p["terminal_embedding.weight"],
                                    p["path_embedding.weight"], p["input_linear.weight"], p["input_layer_norm.weight"],
                                    p["input_layer_norm.bias"], p["attention_parameter"], dropmask=mask)
    pt = {k: torch.from_numpy(v).double() for k, v in p.items()}
    with torch.no_grad():
        _, tcv, tatt = oracle.torch_forward(pt, torch.from_numpy(rec["starts"]), torch.from_numpy(rec["paths"]),
                                            torch.from_numpy(rec["ends"]), torch.from_numpy(rec["label"]),
                                            dropmask=torch.from_numpy(mask).double())
        _, cv0, _ = oracle.torch_forward(pt, torch.from_numpy(rec["starts"]), torch.from_numpy(rec["paths"]),
                                         torch.from_numpy(rec["ends"]), torch.from_numpy(rec["label"]))
    assert np.abs(tcv.numpy() - cv).max() <= 2e-6
    assert np.abs(tatt.numpy() - att).max() <= 2e-6
    assert np.abs(cv0.numpy() - cv).max() > 1e-3          # the mask made a difference


def test_oracle_rejects_out_of_range_index():
    rec = load_golden("tiny")
    bad = rec["starts"].copy()
    bad[0, 0] = rec["opt"]["T"]
    with pytest.raises(IndexError):
        oracle.forward(rec["params"], bad, rec["paths"], rec["ends"], rec["label"])


def test_dropmask_semantics():
    """model.py:60-61: dropout multiplies tanh output before the score AND the weighted sum."""
    rec = load_golden("tiny")
    p = rec["params"]
    B, L = rec["starts"].shape
    H = p["input_linear.weight"].shape[0]
    rng = np.random.default_rng(0)
    mask = (rng.random((B, L, H)) >= 0.25).astype(np.float32) / 0.75
    cv, att, ctx = oracle.encode_forward(rec["starts"], rec["paths"], rec["ends"], p["terminal_embedding.weight"],
                                         p["path_embedding.weight"], p["input_linear.weight"],
                                         p["input_layer_norm.weight"], p["input_layer_norm.bias"],
                                         p["attention_parameter"], dropmask=mask, want_ctx=True)
    cv0, att0, ctx0 = oracle.encode_forward(rec["starts"], rec["paths"], rec["ends"], p["terminal_embedding.weight"],
                                            p["path_embedding.weight"], p["input_linear.weight"],
                                            p["input_layer_norm.weight"], p["input_layer_norm.bias"],
                                            p["attention_parameter"], want_ctx=True)
    assert np.allclose(ctx, ctx0 * mask, atol=1e-7)
    assert np.allclose(cv, (ctx * att[..., None]).sum(1), atol=1e-6)
