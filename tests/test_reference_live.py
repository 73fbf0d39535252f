"""The UNMODIFIED reference modules as the checker (oracle/ref_loader.py: from a reference checkout or from the git-ignored
copy oracle/_ref -- recipe oracle/make_ref.py); at the full sizes of the named configurations the reference's fp64 outputs
are stored under tests/golden/full_size_<cfg>.npz (tests/golden/make_golden_full_size.py), so that comparison needs no
reference tree.

CPU part (``-m "not gpu"``): the restatement oracle/spk_oracle.py against the live reference, and ``convert_model`` on the
reference's shipped trained model (class swap, identical state_dict, fp64 -> fp32 cast).
GPU part: the CUDA path against the reference's fp64 results at the FULL sizes of the named configurations
(cfg2 B=256, cfg3 B=1024 padded, cfg4 8192 atoms), ``convert_model`` end to end (incl. custom nuclear / electronic
embeddings), and the reference's block-level API (PaiNNInteraction / PaiNNMixing / SchNetInteraction forward + gradients).
Tolerance: 1e-5 relative (max-norm) against fp64, BASELINE.json north_star.
"""
import os

import numpy as np
import pytest
import torch

from conftest import rel_err

from oracle import ref_loader as rl

needs_ref = pytest.mark.skipif(not rl.available(), reason="reference modules absent (neither /root/reference nor oracle/_ref)")
TOL = 1e-5


# ------------------------------------------------------------------------------------------------------------ CPU
@needs_ref
def test_oracle_matches_live_reference_cpu():
    from oracle import spk_oracle as O
    from schnetpack_b200 import synthetic as S

    for cfg, kw in (("cfg2", dict(batch=3)), ("cfg1", {}), ("cfg4", dict(n_atoms_total=200))):
        spec, data = S.make_config(cfg, **kw)
        params = S.init_params(spec, seed=2)
        ref = rl.evaluate(rl.build_from_spec(spec, params, torch.float64), data, torch.float64)
        o = O.energy_forces(spec, params, data, dtype=torch.float64)
        assert rel_err(o["energy"].numpy(), ref["energy"].numpy()) < 1e-12
        assert rel_err(o["forces"].numpy(), ref["forces"].numpy()) < 1e-10


@needs_ref
def test_convert_model_swaps_classes_and_keeps_state_dict():
    """INTEGRATION.md section 1: convert_model(reference model) -> CUDA modules with the SAME state_dict (keys and values),
    postprocessors reused, fp64 models cast to fp32 with input casting switched on."""
    import schnetpack_b200 as sb
    from schnetpack_b200 import atomistic, representation
    from schnetpack_b200.model import NeuralNetworkPotential, convert_model

    ref = rl.load_model(rl.testdata("md_ethanol.model"))
    new = convert_model(ref)
    assert isinstance(new, NeuralNetworkPotential) and isinstance(new.representation, representation.PaiNN)
    assert isinstance(new.input_modules[0], atomistic.PairwiseDistances)
    assert isinstance(new.output_modules[0], atomistic.Atomwise) and isinstance(new.output_modules[1], atomistic.Forces)
    assert [type(p).__name__ for p in new.postprocessors] == [type(p).__name__ for p in ref.postprocessors]
    sd0, sd1 = ref.state_dict(), new.state_dict()
    assert list(sd0) == list(sd1)
    for k in sd0:
        assert torch.equal(sd0[k], sd1[k]), k
    assert sorted(new.model_outputs) == sorted(ref.model_outputs)
    assert sorted(new.required_derivatives) == sorted(ref.required_derivatives)
    assert float(new.representation.cutoff) == float(ref.representation.cutoff)     # read by spkdeploy:38
    assert not new.training and not new.cast_inputs
    # fp64 model (spkmd loads every model as fp64 first, md/calculators/schnetpack_calculator.py:98)
    new64 = convert_model(rl.load_model(rl.testdata("md_ethanol.model")).double())
    assert all(p.dtype == torch.float32 for p in new64.parameters()) and new64.cast_inputs
    for k in sd0:
        assert torch.equal(sd0[k].float() if sd0[k].is_floating_point() else sd0[k], new64.state_dict()[k]), k


@needs_ref
def test_convert_model_accepts_shared_blocks_schnet_and_custom_embeddings():
    from schnetpack_b200.model import convert_model

    spk = rl.load()
    emb = spk.nn.embedding
    rep = spk.representation.PaiNN(64, 2, spk.nn.BesselRBF(16, 4.0), spk.nn.CosineCutoff(4.0), shared_interactions=True,
                                   shared_filters=True, nuclear_embedding=emb.NuclearEmbedding(101, 64, zero_init=False),
                                   electronic_embeddings=[emb.ElectronicEmbedding("total_charge", 64, is_charged=True)])
    model = spk.model.NeuralNetworkPotential(rep, input_modules=[spk.atomistic.PairwiseDistances()],
                                             output_modules=[spk.atomistic.Atomwise(n_in=64, output_key="energy"),
                                                             spk.atomistic.Forces()])
    new = convert_model(model)
    assert new.representation.interactions[0] is new.representation.interactions[1]
    assert new.representation.share_filters and type(new.representation.embedding).__name__ == "NuclearEmbedding"
    assert list(model.state_dict()) == list(new.state_dict())
    rep = spk.representation.SchNet(64, 3, spk.nn.GaussianRBF(20, 5.0), spk.nn.CosineCutoff(5.0), n_filters=64)
    model = spk.model.NeuralNetworkPotential(rep, input_modules=[spk.atomistic.PairwiseDistances()],
                                             output_modules=[spk.atomistic.Atomwise(n_in=64, output_key="energy")])
    assert list(model.state_dict()) == list(convert_model(model).state_dict())


# ------------------------------------------------------------------------------------------------------------ GPU
def _cuda_eval(model, data, dev):
    from schnetpack_b200.model import batch_to_device

    x = batch_to_device(data, dev)
    if "_Rij" in x:
        x = model.representation(x)
        x = model.output_modules[0](x)
        res = {"energy": x["energy"]}
    else:
        res = model(x)
    torch.cuda.synchronize()
    return {k: v.detach().cpu().numpy() for k, v in res.items()}


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", ["cfg2", "cfg3", "cfg4"])
def test_full_size_parity_against_reference_on_gpu(cfg):
    """The benchmarked sizes themselves: cfg2 = aspirin x 256 (5376 atoms / 78 k edges, PaiNN E+F), cfg3 = QM9-like x 1024
    with the padded neighbour list (831 488 edge slots, SchNet 128x6, energy), cfg4 = 8192-atom periodic box (PaiNN E+F).
    Checker: the reference's own modules in fp64 on the same inputs and weights (stored, tests/golden/full_size_<cfg>.npz)."""
    from conftest import GOLDEN
    from schnetpack_b200 import synthetic as S
    from schnetpack_b200.model import from_spec

    dev = torch.device("cuda:0")
    spec, data = S.make_config(cfg)
    z = np.load(os.path.join(GOLDEN, f"full_size_{cfg}.npz"))
    assert int(z["n_atoms"]) == data[S.Z].shape[0] and int(z["n_edges"]) == data[S.idx_i].shape[0]
    params = S.init_params(spec, seed=int(z["seed"]))
    out = _cuda_eval(from_spec(spec, params, dev), data, dev)
    ref = {k[6:]: torch.as_tensor(z[k]) for k in z.files if k.startswith("ref64:")}
    e = rel_err(out["energy"], ref["energy"].cpu().numpy())
    print(cfg, "N", data["_atomic_numbers"].shape[0], "E", data["_idx_i"].shape[0], "energy rel err", e)
    assert e < TOL
    if "forces" in out:
        f = rel_err(out["forces"], ref["forces"].cpu().numpy())
        print(cfg, "forces rel err", f)
        assert f < TOL


@pytest.mark.gpu
@needs_ref
def test_convert_model_end_to_end_on_gpu():
    """convert_model(reference trained PaiNN) on the reference's own test geometry: energies / forces (postprocessors on:
    CastTo64 + AddOffsets) equal the reference's to 1e-5 -- and the fp64-loaded model path of spkmd too."""
    from schnetpack_b200 import synthetic as S
    from schnetpack_b200.model import batch_to_device, convert_model

    dev = torch.device("cuda:0")
    data = S.ethanol_batch(4, jitter=0.05, seed=3)
    ref = rl.load_model(rl.testdata("md_ethanol.model")).double().to(dev)
    want = ref({k: (v.double() if v.is_floating_point() else v) for k, v in batch_to_device(data, dev).items()})
    for dtype in (torch.float32, torch.float64):
        src = rl.load_model(rl.testdata("md_ethanol.model")).to(dtype)
        new = convert_model(src).to(dev)
        x = {k: (v.to(dtype) if v.is_floating_point() else v) for k, v in batch_to_device(data, dev).items()}
        got = new(x)
        assert got["forces"].dtype == (torch.float64 if dtype == torch.float64 else got["forces"].dtype)
        for k in ("energy", "forces"):
            err = rel_err(got[k].detach().cpu().numpy(), want[k].detach().cpu().numpy())
            print("convert_model", dtype, k, err)
            assert err < TOL, (dtype, k, err)


@pytest.mark.gpu
@needs_ref
def test_convert_model_custom_embeddings_on_gpu():
    """Models with NuclearEmbedding / ElectronicEmbedding (no ``.weight``; run as given) through convert_model."""
    from schnetpack_b200 import synthetic as S
    from schnetpack_b200.model import batch_to_device, convert_model

    dev = torch.device("cuda:0")
    spk = rl.load()
    emb = spk.nn.embedding
    torch.manual_seed(0)
    rep = spk.representation.PaiNN(128, 2, spk.nn.GaussianRBF(20, 5.0), spk.nn.CosineCutoff(5.0),
                                   nuclear_embedding=emb.NuclearEmbedding(101, 128, zero_init=False),
                                   electronic_embeddings=[emb.ElectronicEmbedding("total_charge", 128, is_charged=True)])
    model = spk.model.NeuralNetworkPotential(rep, input_modules=[spk.atomistic.PairwiseDistances()],
                                             output_modules=[spk.atomistic.Atomwise(n_in=128, output_key="energy"),
                                                             spk.atomistic.Forces()]).eval()
    data = S.aspirin_batch(5, seed=1)
    data["total_charge"] = np.array([0.0, 1.0, -1.0, 2.0, 0.0], dtype=np.float32)
    data["_idx"] = np.arange(5, dtype=np.int64)              # read by ElectronicEmbedding (nn/embedding.py:311)
    new = convert_model(model).to(dev)
    got = new(batch_to_device(data, dev))
    ref = model.double().to(dev)
    want = ref({k: (v.double() if v.is_floating_point() else v) for k, v in batch_to_device(data, dev).items()})
    for k in ("energy", "forces"):
        assert rel_err(got[k].detach().cpu().numpy(), want[k].detach().cpu().numpy()) < TOL, k


@pytest.mark.gpu
@needs_ref
def test_block_level_api_matches_reference_blocks():
    """PaiNNInteraction.forward(q, mu, Wij, dir_ij, idx_i, idx_j, n_atoms), PaiNNMixing.forward(q, mu) and
    SchNetInteraction.forward(x, f_ij, idx_i, idx_j, rcut_ij) called directly, values and first-order gradients, against the
    reference's blocks with the same weights (fp64)."""
    import torch.nn.functional as F_

    from schnetpack_b200 import representation as R
    from schnetpack_b200 import synthetic as S
    from schnetpack_b200.nn import shifted_softplus

    dev = torch.device("cuda:0")
    spk = rl.load()
    b = S.aspirin_batch(4, seed=2)
    ii, jj = torch.as_tensor(b["_idx_i"], device=dev), torch.as_tensor(b["_idx_j"], device=dev)
    N, E, Fd = b["_atomic_numbers"].shape[0], ii.shape[0], 128
    torch.manual_seed(3)

    def leaves(*shapes):
        return [torch.randn(*s, device=dev).requires_grad_() for s in shapes]

    def check(outs, refs, ins, ins64, tol=5e-6):
        seeds = [torch.randn_like(o) for o in outs]
        g = torch.autograd.grad(sum((o * s).sum() for o, s in zip(outs, seeds)), ins)
        g64 = torch.autograd.grad(sum((o * s.double()).sum() for o, s in zip(refs, seeds)), ins64)
        for o, r in zip(outs, refs):
            assert rel_err(o.detach().cpu().numpy(), r.detach().cpu().numpy()) < tol
        for a, r in zip(g, g64):
            assert rel_err(a.cpu().numpy(), r.cpu().numpy()) < 2 * tol

    # --- PaiNNInteraction
    ref_blk = spk.representation.painn.PaiNNInteraction(Fd, F_.silu).to(dev)
    blk = R.PaiNNInteraction(Fd, F_.silu).to(dev).eval()
    blk.load_state_dict(ref_blk.state_dict())
    ins = leaves((N, 1, Fd), (N, 3, Fd), (E, 1, 3 * Fd), (E, 3))
    ins64 = [t.detach().double().requires_grad_() for t in ins]
    outs = blk(*ins, ii, jj, N)
    refs = ref_blk.double()(*ins64, ii, jj, N)
    check(outs, refs, ins, ins64)
    # --- PaiNNMixing
    ref_mix = spk.representation.painn.PaiNNMixing(Fd, F_.silu, 1e-8).to(dev)
    mix = R.PaiNNMixing(Fd, F_.silu, 1e-8).to(dev).eval()
    mix.load_state_dict(ref_mix.state_dict())
    ins = leaves((N, 1, Fd), (N, 3, Fd))
    ins64 = [t.detach().double().requires_grad_() for t in ins]
    check(mix(*ins), ref_mix.double()(*ins64), ins, ins64)
    # --- SchNetInteraction
    ref_s = spk.representation.schnet.SchNetInteraction(Fd, 20, Fd, spk.nn.shifted_softplus).to(dev)
    sblk = R.SchNetInteraction(Fd, 20, Fd, shifted_softplus).to(dev).eval()
    sblk.load_state_dict(ref_s.state_dict())
    x, f_ij = leaves((N, Fd), (E, 20))
    rcut = torch.rand(E, device=dev).requires_grad_()
    ins = [x, f_ij, rcut]
    ins64 = [t.detach().double().requires_grad_() for t in ins]
    out = sblk(x, f_ij, ii, jj, rcut)
    ref = ref_s.double()(ins64[0], ins64[1], ii, jj, ins64[2])
    check([out], [ref], ins, ins64)
