"""The translation between torch.optim.AdamW's state_dict and the flat layout of engine.FlatAdamW (no GPU needed):
a state_dict that goes into the flat buffers and comes back out is the same bit for bit, the state of a parameter
the flat step does not update is carried through, and every state the flat step cannot represent is refused."""
import copy
import io

import pytest
import torch

from coda_neurips2023_b200.engine import (FlatParameters, _no_decay, adamw_flat_index, adamw_hyperparameters,
                                          adamw_numbered_state, adamw_state_to_flat, bind_adamw_state)


def _model():
    torch.manual_seed(0)
    return torch.nn.ModuleDict({"enc": torch.nn.Linear(5, 70), "norm": torch.nn.LayerNorm(70),
                                "out": torch.nn.Linear(70, 3), "unused": torch.nn.Linear(70, 2)})


def _adamw(model, filter_biases_wd, **kw):
    """the reference's build_optimizer (optimizer.py:5-36)"""
    decay, no_decay = [], []
    for name, p in model.named_parameters():
        (no_decay if filter_biases_wd and _no_decay(name, p) else decay).append(p)
    if filter_biases_wd:
        groups = [{"params": no_decay, "weight_decay": 0.0}, {"params": decay, "weight_decay": 0.1}]
    else:
        groups = [{"params": decay, "weight_decay": 0.1}]
    return torch.optim.AdamW(groups, lr=1e-2, **kw)


def _train(model, opt, steps, with_unused):
    g = torch.Generator().manual_seed(steps)
    for _ in range(steps):
        opt.zero_grad()
        h = model["norm"](model["enc"](torch.randn(4, 5, generator=g)))
        loss = model["out"](h).pow(2).mean()
        if with_unused:
            loss = loss + model["unused"](h).pow(2).mean()
        loss.backward()
        opt.step()


def _layout(model):
    """flat layout in a different order than the optimizer's (as TrainStep lays it out in gradient-ready order), the
    parameter that receives no gradient last and inactive"""
    params = [p for n, p in model.named_parameters() if not n.startswith("unused")][::-1]
    params += list(model["unused"].parameters())
    flat = FlatParameters(model, order=params)
    active = [not n.startswith("unused") for n in flat.names]
    return flat, active


def _bits(t):
    return t.detach().reshape(-1).view(torch.int32)


def _assert_same_state_dict(got, exp):
    assert got["param_groups"] == exp["param_groups"]
    assert sorted(got["state"]) == sorted(exp["state"])
    for k, st in exp["state"].items():
        assert sorted(got["state"][k]) == sorted(st), k
        for key, t in st.items():
            g = got["state"][k][key]
            assert g.dtype == t.dtype and g.shape == t.shape and g.device == t.device, (k, key)
            assert torch.equal(_bits(g), _bits(t)), (k, key)


@pytest.mark.parametrize("filter_biases_wd", [False, True])
def test_state_dict_round_trip_through_the_flat_layout_is_bit_exact(filter_biases_wd):
    model = _model()
    opt = _adamw(model, filter_biases_wd)
    _train(model, opt, 2, with_unused=True)      # the unused head had a gradient once (a stage-1 run, say)...
    _train(model, opt, 3, with_unused=False)     # ...and not since: its state stays at step 2
    sd = copy.deepcopy(opt.state_dict())
    flat, active = _layout(model)
    index = adamw_flat_index(opt, flat)
    exp_avg, exp_avg_sq = torch.zeros_like(flat.flat_grad), torch.zeros_like(flat.flat_grad)
    step, carried = adamw_state_to_flat(sd["state"], index, flat, active, exp_avg, exp_avg_sq)
    assert step == 5.0
    assert carried == {i: 2.0 for i, a in enumerate(active) if not a}
    for i, p in enumerate(flat.params):
        off = flat.offsets[i]
        assert torch.equal(exp_avg[off:off + p.numel()], sd["state"][index[i]]["exp_avg"].reshape(-1))
    bind_adamw_state(opt, index, flat, active, exp_avg, exp_avg_sq, step, carried)
    out = opt.state_dict()
    _assert_same_state_dict(out, sd)
    for i, p in enumerate(flat.params):        # the optimizer's moments are views of the flat buffers
        assert opt.state[p]["exp_avg"].data_ptr() == exp_avg[flat.offsets[i]:].data_ptr()
    # what torch.save writes of the views loads into a stock AdamW as the same state
    buf = io.BytesIO()
    torch.save({"optimizer": out}, buf)
    buf.seek(0)
    model2 = _model()
    opt2 = _adamw(model2, filter_biases_wd)
    opt2.load_state_dict(torch.load(buf, map_location="cpu")["optimizer"])
    _assert_same_state_dict(opt2.state_dict(), sd)
    # the stock optimizer steps it as it would have stepped its own
    ref = _model()
    ref.load_state_dict(model.state_dict())
    model2.load_state_dict(model.state_dict())
    ref_opt = _adamw(ref, filter_biases_wd)
    ref_opt.load_state_dict(copy.deepcopy(sd))
    _train(ref, ref_opt, 2, with_unused=False)
    _train(model2, opt2, 2, with_unused=False)
    for (n, p), q in zip(ref.named_parameters(), model2.parameters()):
        assert torch.equal(p, q), n


def test_reloading_its_own_state_in_memory_keeps_the_moments():
    """After binding, the optimizer's moments are views of the flat buffers, and torch's load_state_dict keeps a
    tensor that is already on the right device: importing again reads the buffers it writes."""
    model = _model()
    opt = _adamw(model, True)
    _train(model, opt, 3, with_unused=True)
    sd = copy.deepcopy(opt.state_dict())
    flat, active = _layout(model)
    index = adamw_flat_index(opt, flat)
    exp_avg, exp_avg_sq = torch.zeros_like(flat.flat_grad), torch.zeros_like(flat.flat_grad)
    step, carried = adamw_state_to_flat(adamw_numbered_state(opt), index, flat, active, exp_avg, exp_avg_sq)
    bind_adamw_state(opt, index, flat, active, exp_avg, exp_avg_sq, step, carried)
    m0, v0 = exp_avg.clone(), exp_avg_sq.clone()
    opt.load_state_dict(opt.state_dict())
    assert opt.state[flat.params[0]]["exp_avg"].data_ptr() == exp_avg.data_ptr() + 4 * flat.offsets[0]
    step2, carried2 = adamw_state_to_flat(adamw_numbered_state(opt), index, flat, active, exp_avg, exp_avg_sq)
    assert (step2, carried2) == (step, carried)
    assert torch.equal(_bits(exp_avg), _bits(m0)) and torch.equal(_bits(exp_avg_sq), _bits(v0))
    assert m0.abs().sum() > 0
    bind_adamw_state(opt, index, flat, active, exp_avg, exp_avg_sq, step2, carried2)
    _assert_same_state_dict(opt.state_dict(), sd)


def test_fresh_optimizer_adopts_step_zero_and_exports_no_state():
    model = _model()
    opt = _adamw(model, True)
    sd = copy.deepcopy(opt.state_dict())
    flat, active = _layout(model)
    index = adamw_flat_index(opt, flat)
    exp_avg, exp_avg_sq = torch.ones_like(flat.flat_grad), torch.ones_like(flat.flat_grad)
    step, carried = adamw_state_to_flat(adamw_numbered_state(opt), index, flat, active, exp_avg, exp_avg_sq)
    assert step == 0.0 and carried == {}
    assert not exp_avg.any() and not exp_avg_sq.any()
    bind_adamw_state(opt, index, flat, active, exp_avg, exp_avg_sq, step, carried)
    _assert_same_state_dict(opt.state_dict(), sd)


@pytest.mark.parametrize("filter_biases_wd", [False, True])
def test_hyperparameters_come_from_the_param_groups(filter_biases_wd):
    model = _model()
    opt = _adamw(model, filter_biases_wd, betas=(0.8, 0.99), eps=1e-7)
    flat, _ = _layout(model)
    wds, betas, eps = adamw_hyperparameters(opt.param_groups, adamw_flat_index(opt, flat))
    assert betas == (0.8, 0.99) and eps == 1e-7
    assert wds == [0.0 if filter_biases_wd and _no_decay(n, p) else 0.1 for n, p in zip(flat.names, flat.params)]
    opt.param_groups[-1]["betas"] = (0.9, 0.999)
    if filter_biases_wd:
        with pytest.raises(ValueError, match="betas"):
            adamw_hyperparameters(opt.param_groups, adamw_flat_index(opt, flat))


def test_optimizer_over_other_parameters_is_refused():
    model = _model()
    short = torch.optim.AdamW([p for n, p in model.named_parameters() if n != "norm.weight"])
    extra = torch.optim.AdamW(list(model.parameters()) + [torch.nn.Parameter(torch.zeros(3))])
    flat, _ = _layout(model)
    with pytest.raises(ValueError, match=r"not in the optimizer: norm\.weight"):
        adamw_flat_index(short, flat)
    with pytest.raises(ValueError, match="1 optimizer parameters that are not trainable parameters"):
        adamw_flat_index(extra, flat)
    with pytest.raises(ValueError, match="SGD"):
        adamw_flat_index(torch.optim.SGD(model.parameters(), lr=0.1), flat)


@pytest.mark.parametrize("option", ["amsgrad", "maximize", "differentiable"])
def test_options_that_change_the_update_rule_are_refused(option):
    model = _model()
    opt = _adamw(model, True, **{option: True})
    flat, _ = _layout(model)
    with pytest.raises(ValueError, match=option):
        adamw_hyperparameters(opt.param_groups, adamw_flat_index(opt, flat))


def _trained_state():
    model = _model()
    opt = _adamw(model, True)
    _train(model, opt, 3, with_unused=False)
    flat, active = _layout(model)
    index = adamw_flat_index(opt, flat)
    return flat, active, index, copy.deepcopy(opt.state_dict()["state"])


def test_mixed_step_counts_are_refused():
    flat, active, index, state = _trained_state()
    state[index[1]]["step"] = torch.tensor(7.0)
    buf = torch.full_like(flat.flat_grad, 3.0)
    with pytest.raises(ValueError, match=rf"different AdamW step counts \(.*{flat.names[1]}: 7"):
        adamw_state_to_flat(state, index, flat, active, buf, buf.clone())
    assert (buf == 3.0).all(), "a refused state must leave the flat buffers alone"


def test_state_on_some_active_parameters_only_is_refused():
    flat, active, index, state = _trained_state()
    del state[index[0]]
    with pytest.raises(ValueError, match=rf"without: {flat.names[0]}"):
        adamw_state_to_flat(state, index, flat, active, torch.zeros_like(flat.flat_grad),
                            torch.zeros_like(flat.flat_grad))


def test_state_without_a_step_count_is_refused():
    flat, active, index, state = _trained_state()
    del state[index[2]]["step"]
    with pytest.raises(ValueError, match=rf"{flat.names[2]} has no step count"):
        adamw_state_to_flat(state, index, flat, active, torch.zeros_like(flat.flat_grad),
                            torch.zeros_like(flat.flat_grad))


def test_moments_that_do_not_fit_the_parameter_are_refused():
    flat, active, index, state = _trained_state()
    state[index[0]]["exp_avg"] = torch.zeros(2)
    with pytest.raises(ValueError, match=rf"{flat.names[0]}: exp_avg \(2,\) does not fit"):
        adamw_state_to_flat(state, index, flat, active, torch.zeros_like(flat.flat_grad),
                            torch.zeros_like(flat.flat_grad))
