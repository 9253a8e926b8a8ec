"""CPU: the ActionValue approximator (apprfunc/mlp.py, reference mlp.py:224-245) registers as `mlp_ActionValue`, keeps
the reference's state_dict keys and action_distribution_cls, and refuses output activations its kernels do not run."""
import pytest


def _kwargs(**over):
    kw = dict(apprfunc="MLP", name="ActionValue", obs_dim=6, act_dim=1, hidden_sizes=[256, 256, 256],
              hidden_activation="relu", output_activation="linear", action_distribution_cls="dist")
    kw.update(over)
    return kw


def test_action_value_keys_and_shape():
    from gops_b200.create_pkg.create_apprfunc import create_apprfunc
    q = create_apprfunc(**_kwargs())
    assert list(q.state_dict()) == [f"q.{j}.{w}" for j in (0, 2, 4, 6) for w in ("weight", "bias")]
    assert tuple(q.q[0].weight.shape) == (256, 7) and tuple(q.q[6].weight.shape) == (1, 256)
    assert q.action_distribution_cls == "dist"


def test_action_value_refuses_a_nonlinear_output():
    from gops_b200.create_pkg.create_apprfunc import create_apprfunc
    with pytest.raises(NotImplementedError, match="linear"):
        create_apprfunc(**_kwargs(output_activation="tanh"))
