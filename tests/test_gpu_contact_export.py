"""GPU: the exported `Contacts` arrays, element by element in export order, against the CPU oracle.

The export writes each environment's contacts behind those of all earlier environments.  Its offsets are sums of the contact
counts the collide kernel leaves per CTA and per environment: summed by the export itself up to 8192 environments, scanned by
a separate kernel above.  Both paths are pinned here, with the last export CTA partly filled, and so is the overflow rule (a
buffer smaller than the contact count: the count keeps growing and the contacts past the capacity are dropped).
"""

import functools

import numpy as np
import pytest
import torch

import newton_b200
from newton_b200 import scenes

pytestmark = pytest.mark.gpu

FIELDS = ("shape0", "shape1", "point0", "point1", "offset0", "offset1", "normal", "margin0", "margin1")


def _quadrupeds_on_ground(envs):
    model = scenes.quadruped_model(envs, seed=1)
    model.joint_q.view(envs, -1)[:, 2] = 0.45  # every foot within the contact gap of the ground
    scenes.host_fk(model, model.joint_q, model.joint_qd, model)
    return model


@functools.lru_cache(maxsize=None)
def _case(envs):
    """The settled scene and the oracle's contacts (reference sort-key order) stably re-ordered by environment: the export's
    (env, key) order."""
    import oracle

    model = _quadrupeds_on_ground(envs)
    pipe = oracle.CollisionPipeline(model)
    c = pipe.contacts()
    pipe.collide(model.state(), c)
    n = int(c.rigid_contact_count.item())
    arrays = {k: getattr(c, "rigid_contact_" + k)[:n].numpy() for k in FIELDS}
    world = model.shape_world.numpy()
    env = np.maximum(world[arrays["shape0"]], world[arrays["shape1"]])
    order = np.argsort(env, kind="stable")
    return model, n, {k: v[order] for k, v in arrays.items()}


@pytest.mark.parametrize("envs", [300, 4096, 8200])
def test_export_offsets_match_oracle(oracle_lib, cuda_lib, envs):
    """300 / 4096 environments: offsets summed by the export kernel (1- and 8-warp collide CTAs); 8200: the scan path."""
    model, n, ref = _case(envs)
    mg = model.to("cuda:0")
    pipe = newton_b200.CollisionPipeline(mg)
    c = pipe.contacts()
    pipe.collide(mg.state(), c)
    torch.cuda.synchronize()
    assert n > 4 * envs
    assert int(c.rigid_contact_count.item()) == n
    for k in FIELDS:
        np.testing.assert_array_equal(getattr(c, "rigid_contact_" + k)[:n].cpu().numpy(), ref[k], err_msg=k)


@pytest.mark.parametrize("envs", [4096, 8200])
def test_export_overflow_drops_the_tail(oracle_lib, cuda_lib, envs):
    """A buffer that holds about 60 % of the contacts: the count is the full count and the buffer holds the first contacts in
    export order."""
    model, n, ref = _case(envs)
    cap = (n * 3) // 5 + 7  # not a multiple of an environment's or a CTA's contacts
    mg = model.to("cuda:0")
    pipe = newton_b200.CollisionPipeline(mg, rigid_contact_max=cap)
    c = pipe.contacts()
    assert c.rigid_contact_max == cap
    pipe.collide(mg.state(), c)
    torch.cuda.synchronize()
    assert int(c.rigid_contact_count.item()) == n
    for k in FIELDS:
        np.testing.assert_array_equal(getattr(c, "rigid_contact_" + k)[:cap].cpu().numpy(), ref[k][:cap], err_msg=k)
