"""The fused training steps' optimizer state in torch.optim.Adam's format (wav2lip_b200/training.py): the conversion between
`torch.optim.Adam([p for p in model.parameters() if p.requires_grad], lr, betas).state_dict()` (state keyed by the index
into that list) and the by-name form the native Adam is addressed with.  CPU only: the mirrors' parameters on the host."""
import copy

import pytest
import torch

from wav2lip_b200.models import SyncNet_color, Wav2Lip, Wav2Lip_disc_qual
from wav2lip_b200.training import adam_param_names, adam_state_from_named, adam_state_to_named


def _stepped_adam(module, betas, steps, seed):
    params = [p for p in module.parameters() if p.requires_grad]
    opt = torch.optim.Adam(params, lr=1e-4, betas=betas)
    g = torch.Generator().manual_seed(seed)
    for _ in range(steps):
        for p in params:
            p.grad = torch.randn(p.shape, generator=g)
        opt.step()
    return params, opt


def _assert_same_state(a, b):
    assert a["param_groups"] == b["param_groups"]
    assert list(a["state"].keys()) == list(b["state"].keys())
    for i in a["state"]:
        for k in ("step", "exp_avg", "exp_avg_sq"):
            assert torch.equal(a["state"][i][k], b["state"][i][k]), (i, k)


@pytest.mark.parametrize("net, betas", [(Wav2Lip, (0.5, 0.999)), (Wav2Lip_disc_qual, (0.5, 0.999)), (SyncNet_color, (0.9, 0.999))])
def test_adam_state_dict_round_trips_through_the_named_form(net, betas):
    torch.manual_seed(0)
    module = net()
    names = adam_param_names(module)
    assert names == [n for n, _ in module.named_parameters()]      # every mirror parameter trains
    params, opt = _stepped_adam(module, betas, steps=2, seed=1)
    sd = opt.state_dict()
    named = adam_state_to_named(sd, names)
    assert named["step"] == 2 and set(named["exp_avg"]) == set(names)
    i = len(names) // 2
    assert named["exp_avg"][names[i]] is sd["state"][i]["exp_avg"]     # index i is the i-th parameter by name
    back = adam_state_from_named(named, names)
    _assert_same_state(back, sd)
    # loadable: a fresh optimizer over the same list takes it, and steps exactly as the original does
    fresh = torch.optim.Adam(params, lr=1e-4, betas=betas)
    fresh.load_state_dict(copy.deepcopy(back))        # (load_state_dict keeps the tensors it is given)
    _assert_same_state(fresh.state_dict(), sd)
    before = [p.detach().clone() for p in params]
    g = torch.Generator().manual_seed(7)
    grads = [torch.randn(p.shape, generator=g) for p in params]
    for p, gr in zip(params, grads):
        p.grad = gr.clone()
    opt.step()
    after_orig = [p.detach().clone() for p in params]
    with torch.no_grad():
        for p, b0 in zip(params, before):
            p.copy_(b0)
    for p, gr in zip(params, grads):
        p.grad = gr.clone()
    fresh.step()
    for a, p in zip(after_orig, params):
        assert torch.equal(a, p.detach())


def test_adam_state_before_any_step_is_empty_and_step_zero():
    module = Wav2Lip_disc_qual()
    names = adam_param_names(module)
    sd = torch.optim.Adam(list(module.parameters()), lr=1e-4, betas=(0.5, 0.999)).state_dict()
    named = adam_state_to_named(sd, names)
    assert named["step"] == 0 and named["exp_avg"] == {}
    _assert_same_state(adam_state_from_named(named, names), sd)


def test_adam_state_rejects_a_foreign_layout():
    module = Wav2Lip_disc_qual()
    names = adam_param_names(module)
    _, opt = _stepped_adam(module, (0.5, 0.999), steps=1, seed=2)
    sd = opt.state_dict()
    with pytest.raises(ValueError):
        adam_state_to_named(sd, names[:-1])                 # a different parameter list
    bad = {"state": dict(sd["state"]), "param_groups": sd["param_groups"]}
    bad["state"][0] = dict(bad["state"][0], step=torch.tensor(5.0))
    with pytest.raises(ValueError):
        adam_state_to_named(bad, names)                     # two step counts in one optimizer
    with pytest.raises(ValueError):
        adam_state_from_named({"step": 1, "exp_avg": {"nope": torch.zeros(1)}, "exp_avg_sq": {}, "param_groups": []}, names)
