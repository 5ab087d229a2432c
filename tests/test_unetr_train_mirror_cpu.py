"""CPU checks of the UNETR decoder's device mirror (tests/unetr_train_mirror.py): without rounding it is the float64
training-mode restatement (tests/unetr_train_ref.py); with rounding, float32 against float64 measures the flip noise the device
shows against the mirror; and faults planted in the mirror show what the slope bounds of tests/test_gpu_unetr_train_mirror.py
catch that twice the noise floor (tests/test_gpu_unetr_train.py::test_decoder_backward_against_float64) lets through."""
import pytest
import torch

from oracle import unetr_ref
from tests import unetr_train_mirror as mirror
from tests import unetr_train_noise_floor as nf
from tests import unetr_train_ref as ref


@pytest.mark.parametrize("plan", sorted(nf.CASES))
def test_mirror_without_rounding_is_the_float64_restatement(plan):
    kw, _ = nf.CASES[plan]
    sd = mirror.device_weights(unetr_ref.seeded_state(seed=nf.STATE_SEED, **kw))
    g = torch.Generator().manual_seed(9)
    z = mirror.bf(torch.randn(2, 64, 4, 4, generator=g))
    dm = torch.randn(2, 3, 64, 64, generator=g)
    lv = ref.leaves(sd)
    zz = z.double().requires_grad_(True)
    want = ref.forward_maps(lv, zz, train=True)
    (want * dm.double()).sum().backward()
    got, maps, running = mirror.run(sd, z, dm, torch.float64, rounding=False)
    assert float((maps - want.detach()).abs().max()) < 1e-10
    assert ref.rel_l2(got["d_embedding"], zz.grad) < 1e-10
    keys = [k for k, v in lv.items() if isinstance(v, torch.Tensor) and v.requires_grad]
    assert set(got) == set(keys) | {"d_embedding"}
    zero = mirror.zero_grad_keys(keys)
    big = max(float(lv[k].grad.norm()) for k in keys if k not in zero)
    for k in keys:
        if k in zero:   # rounding noise on both sides
            assert float((got[k] - lv[k].grad).norm()) < 1e-10 * big, k
        else:
            assert ref.rel_l2(got[k], lv[k].grad) < 1e-10, k
    assert set(running) == {k for k in lv if k.endswith(("running_mean", "running_var"))}
    for k, v in running.items():
        assert float((v - lv[k]).abs().max()) < 1e-12, k
        assert not torch.equal(v, sd[k].double()), k


@pytest.fixture(scope="module")
def interp():
    """the reduced bilinear case of the GPU tests: the float64 restatement, the float64 and float32 mirrors, the noise floor"""
    sd, z, dm = nf.case_inputs("interp")
    r64, _, _ = mirror.run(sd, z, dm, torch.float64, rounding=False)
    m64, _, run64 = mirror.run(sd, z, dm, torch.float64)
    m32, _, run32 = mirror.run(sd, z, dm, torch.float32)
    zero = mirror.zero_grad_keys(r64)
    floor = {k: ref.rel_l2(m32[k], r64[k]) for k in r64 if k not in zero}
    return dict(sd=sd, z=z, dm=dm, r64=r64, m64=m64, run64=run64, m32=m32, run32=run32, floor=floor)


def mirror_verdict(got, running, c):
    """(tensors outside their family's slope / rel-L2 bound, largest running-statistics difference) against the float64 mirror"""
    bounds = mirror.GRAD_BOUNDS
    out = {}
    for k in c["floor"]:
        if k == "d_embedding":
            continue
        r, s = ref.rel_l2(got[k], c["m64"][k]), abs(mirror.slope(got[k], c["m64"][k]) - 1)
        tol = bounds[mirror.family(k)]
        if not (r <= tol[0] and s <= tol[1]):
            out[k] = (r, s, tol)
    return out, max(float((running[k].double() - c["run64"][k]).abs().max()) for k in running)


def floor_verdict(got, c):
    """tensors at or past twice their noise floor against the float64 restatement"""
    return {k: ref.rel_l2(got[k], c["r64"][k]) / c["floor"][k] for k in c["floor"] if not ref.rel_l2(got[k], c["r64"][k]) < 2 * c["floor"][k]}


def test_float32_flip_noise(interp):
    """float32 against float64, both rounding where the device rounds: the distance the device sits at from the mirror.  Per
    tensor the slope moves far less than rel-L2, and the float32 mirror passes the reduced plans' bounds as the device does."""
    c = interp
    fam = {}
    for k in c["floor"]:
        r, s = ref.rel_l2(c["m32"][k], c["m64"][k]), abs(mirror.slope(c["m32"][k], c["m64"][k]) - 1)
        f = fam.setdefault("d_embedding" if k == "d_embedding" else mirror.family(k), [0.0, 0.0])
        f[0], f[1] = max(f[0], r), max(f[1], s)
    print("float32 against float64 mirror, worst (rel-L2, |slope - 1|) per family:", fam)
    bad, running = mirror_verdict(c["m32"], c["run32"], c)
    assert not bad, bad
    assert running < mirror.TOL_RUNNING
    assert all(f[1] < f[0] / 3 for f in fam.values())


# (fault, whether twice the noise floor lets it through): wgrad x 1.05 rather than 1.02, as the slope noise of the reduced plan's
# 3x3 weights reaches 1.4e-2 (a 2 % scaling is out of reach end to end, see tests/test_gpu_unetr_train_mirror.py)
FAULTS = [("wgrad_scale:decoder.blocks.1.block.1.weight:1.05", True),
          ("bn_biased_var", True),
          ("in_no_mean:decoder_head.block.0", False),
          ("drop_skip:decoder.blocks.0", False)]


@pytest.mark.parametrize("fault,floor_misses", FAULTS)
def test_planted_fault_is_caught_by_the_mirror_bounds(interp, fault, floor_misses):
    c = interp
    got, _, running = mirror.run(c["sd"], c["z"], c["dm"], torch.float32, faults=[fault])
    bad, run_err = mirror_verdict(got, running, c)
    print(fault, "outside the mirror bounds:", sorted(bad), "running", run_err, "at 2x floor or past:", floor_verdict(got, c))
    assert bad or run_err >= mirror.TOL_RUNNING
    assert (not floor_verdict(got, c)) == floor_misses
