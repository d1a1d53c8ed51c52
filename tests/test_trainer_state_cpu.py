"""Parameter and optimiser state of both stage-1 trainers against the oracle, on the host: the initialisation's
random stream, the state-dict keys and shapes of every network, and the torch.optim.Adam state-dict schema of the
checkpoint in both directions.  The trainers are built with device="cpu" (their layout calls are host-only);
no kernel runs."""
import pytest
import torch

from b200 import atlas as A
from b200 import seg as SG
from csrc_build import ensure_built
from oracle import atlas_oracle as O
from oracle import seg_oracle as S

PE_MAPPING = dict(use_positional_encoding_mapping1=True, number_of_positional_encoding_mapping1=4)


@pytest.fixture(scope="module", autouse=True)
def _built():
    ensure_built()


class Atlas:
    """AtlasTrainer and the oracle networks of src/stage1_neural_atlas.py, keyed by the trainer's network names."""

    def __init__(self, config=None):
        self.config = config
        pe = A.mapping_pe_freqs(config)
        self.specs = dict(mapping=O.MlpSpec(3, 2, 256, True, pe, (), 6) if pe else O.MAPPING_SPEC, atlas=O.ATLAS_SPEC)

    def trainer(self):
        return A.AtlasTrainer(None, self.config, device="cpu")

    def init_nets(self):
        """The script's construction order: mapping, then atlas."""
        return dict(mapping=O.init_mlp(self.specs["mapping"]), atlas=O.init_mlp(self.specs["atlas"]))

    def make_optimizer(self, nets):
        return O.make_optimizer(nets["mapping"], nets["atlas"])

    def load_state(self, tr, nets):
        tr.load_state(O.state_dict_of(nets["mapping"]), O.state_dict_of(nets["atlas"]))


class Seg:
    """SegTrainer and the oracle networks of src/stage1_neural_atlas_seg.py."""
    specs = dict(mapping1=S.MAPPING1_SPEC, mapping2=S.MAPPING2_SPEC, alpha=S.ALPHA_SPEC, atlas=S.ATLAS_SPEC)

    def trainer(self):
        return SG.SegTrainer(None, None, None, device="cpu")

    def init_nets(self):
        return S.init_nets()

    def make_optimizer(self, nets):
        return S.make_optimizer(nets)

    def load_state(self, tr, nets):
        tr.load_state({k: O.state_dict_of(v) for k, v in nets.items()})


KINDS = {"atlas": Atlas(), "atlas_pe4": Atlas(PE_MAPPING), "seg": Seg()}
GROUP_ORDER = {"atlas": ("mapping", "atlas"), "atlas_pe4": ("mapping", "atlas"),
               "seg": ("mapping1", "mapping2", "alpha", "atlas")}          # the reference's optimiser groups


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("seed", [0, 1234])
def test_init_like_reference_is_the_oracle_init(kind, seed):
    k = KINDS[kind]
    tr = k.trainer()
    torch.manual_seed(seed)
    tr.init_like_reference()
    torch.manual_seed(seed)
    nets = k.init_nets()
    assert set(nets) == set(GROUP_ORDER[kind])
    for which, params in nets.items():
        ref = O.state_dict_of(params)
        got = tr.state_dict(which)
        assert list(got) == list(ref), which
        for name in ref:
            assert got[name].dtype == torch.float32
            assert torch.equal(got[name], ref[name]), (which, name)


@pytest.mark.parametrize("kind", KINDS)
def test_state_dict_keys_shapes_and_round_trip(kind):
    k = KINDS[kind]
    tr = k.trainer()
    for which, spec in k.specs.items():
        got = tr.state_dict(which)
        assert [(n, tuple(v.shape)) for n, v in got.items()] == \
            [(n, tuple(v.shape)) for n, v in O.state_dict_of(O.init_mlp(spec)).items()], which
    torch.manual_seed(5)
    nets = k.init_nets()
    k.load_state(tr, nets)
    for which, params in nets.items():
        for (name, got), ref in zip(tr.state_dict(which).items(), params):
            assert torch.equal(got, ref), (which, name)
    # every parameter lands in its own place: the networks' views tile their slices of the flat buffer
    assert sum(p.numel() for ps in nets.values() for p in ps) == \
        sum(v.numel() for w in GROUP_ORDER[kind] for v in tr.param_views(w).values())


def _adam_steps(opt, nets, n, seed):
    g = torch.Generator().manual_seed(seed)
    for _ in range(n):
        for params in nets.values():
            for p in params:
                p.grad = torch.randn(p.shape, generator=g)
        opt.step()


@pytest.mark.parametrize("kind", KINDS)
def test_optimizer_state_dict_matches_torch_adam(kind):
    k = KINDS[kind]
    tr = k.trainer()
    torch.manual_seed(3)
    nets = {w: [p.requires_grad_(True) for p in ps] for w, ps in k.init_nets().items()}
    opt = k.make_optimizer(nets)
    _adam_steps(opt, nets, 2, seed=11)
    ref = opt.state_dict()
    tr.load_optimizer_state_dict(ref)
    assert int(tr.step_count) == 2
    got = tr.optimizer_state_dict()

    assert list(got["state"]) == list(ref["state"])
    for i, r in ref["state"].items():
        s = got["state"][i]
        assert set(s) == set(r), i
        for key in ("step", "exp_avg", "exp_avg_sq"):
            assert s[key].dtype == r[key].dtype and s[key].shape == r[key].shape, (i, key)
            assert torch.equal(s[key], r[key]), (i, key)
    assert len(got["param_groups"]) == len(ref["param_groups"]) == len(GROUP_ORDER[kind])
    for which, g, r in zip(GROUP_ORDER[kind], got["param_groups"], ref["param_groups"]):
        assert g["params"] == r["params"], which
        assert len(g["params"]) == len(nets[which]), which
        for key in ("lr", "betas", "eps", "weight_decay"):
            assert g[key] == r[key], (which, key)
        # the exported groups carry a subset of torch's keys (torch adds decoupled_weight_decay), no key of their own
        assert set(g) <= set(r), (which, set(g) - set(r))

    # the exported dict loads into the oracle's optimiser, which then takes a step
    torch.manual_seed(3)
    nets2 = {w: [p.requires_grad_(True) for p in ps] for w, ps in k.init_nets().items()}
    opt2 = k.make_optimizer(nets2)
    opt2.load_state_dict(got)
    before = [p.detach().clone() for ps in nets2.values() for p in ps]
    _adam_steps(opt2, nets2, 1, seed=12)
    for i, s in opt2.state_dict()["state"].items():
        assert float(s["step"]) == 3.0, i
    assert any(not torch.equal(b, p.detach()) for b, p in zip(before, (p for ps in nets2.values() for p in ps)))

