"""The initial weights of every model class: what `init_weights(seed)` draws, and so what a model built with `seed=` holds.

No GPU: a CPU stand-in for the C-ABI answers the calls a host class makes while it is built (`vb_create` / `vb_create_<kind>`,
`vb_num_weights`, `vb_weight_info`, `vb_set_weight`, `vb_finalize`, `vb_destroy`) with the weight list the engine gives that
configuration.  Where an oracle restates the reference's initialisers (oracle/weights.py, tests/*_oracle.py), the weights must
equal its `init_weights(cfg, seed)` bit for bit.  The small-dataset ViT, MAE and SimMIM have no such oracle (their oracles draw
test weights of another scale), so their weights are pinned by digest."""
import hashlib

import pytest

import ats_oracle
import cases
import cct_oracle
import crossformer_oracle
import cvt_oracle
import levit_oracle
import mim_oracle
import mobilevit_oracle
import nest_oracle
import oracle
import pit_oracle
import regionvit_oracle
import scalable_vit_oracle
import small_vit_oracle
import twins_oracle
from oracle.weights import _vit_layer
import vit_tensorflow_b200 as vb
from vit_tensorflow_b200 import _lib

SEEDS = (0, 1)
FAMILY_ORACLES = (cct_oracle, levit_oracle, cvt_oracle, twins_oracle, crossformer_oracle, nest_oracle, regionvit_oracle, mobilevit_oracle,
                  scalable_vit_oracle, pit_oracle)


class _SpecEngine:
    """The C-ABI calls of building a model, answered from `specs`: kind name -> [(weight name, shape)] in the engine's order."""

    def __init__(self, specs):
        self.specs, self.handles = specs, []

    def __getattr__(self, name):
        if name.startswith("vb_create"):            # vb_create(cfg, device, &h) and vb_create_<kind>(cfg, ext, device, &h)
            return self._create
        raise AttributeError(name)

    def _create(self, cfg_ref, *rest):
        kind = {v: k for k, v in _lib.KIND.items()}[cfg_ref._obj.kind]
        self.handles.append(list(self.specs[kind]))
        rest[-1]._obj.value = len(self.handles)
        return 0

    def _list(self, h):
        return self.handles[(h.value if hasattr(h, "value") else h) - 1]

    def vb_num_weights(self, h):
        return len(self._list(h))

    def vb_weight_info(self, h, i, name_ref, shape, ndim_ref):
        name, shp = self._list(h)[i]
        name_ref._obj.value = name.encode()
        for j, d in enumerate(shp):
            shape[j] = d
        ndim_ref._obj.value = len(shp)
        return 0

    def vb_set_weight(self, h, name, ptr, shape, ndim):
        return 0

    def vb_finalize(self, h):
        return 0

    def vb_destroy(self, h):
        pass


def _names(oracle_specs):
    """[(name, shape)] of an oracle's weight_specs (name -> (shape, initialiser))."""
    return [(n, tuple(s)) for n, (s, _) in oracle_specs.items()]


def _vit_cfg(c, depth):
    return oracle.make_config("vit", image_size=c["image"], patch_size=c["patch"], num_classes=5, dim=c["dim"], depth=depth,
                              heads=c["heads"], mlp_dim=c["mlp_dim"], dim_head=c["dim_head"])


def _oracle_cases():
    """id -> (specs by kind, build(seed), expected(seed))."""
    out = {}
    for name in cases.SMALL:
        cfg = cases.cfg_of(name)
        out[f"{cfg['kind']}:{name}"] = ({cfg["kind"]: _names(oracle.weight_specs(cfg))},
                                        lambda seed, cfg=cfg: vb.from_config(cfg, seed=seed),
                                        lambda seed, cfg=cfg: oracle.init_weights(cfg, seed))
    for cls, name in ((vb.DistillableViT, "vit_small"), (vb.DistillableT2TViT, "t2t_small")):
        cfg, kw = cases.cfg_of(name), {k: v for k, v in cases.SMALL[name].items() if k != "kind"}
        out[f"{cls.__name__}:{name}"] = ({cfg["kind"]: _names(oracle.weight_specs(cfg))},
                                         lambda seed, cls=cls, kw=kw: cls(**kw, seed=seed),
                                         lambda seed, cfg=cfg: oracle.init_weights(cfg, seed))
    # an injected transformer: the engine holds the embedding and the head only (no layers)
    shell = oracle.make_config("vit", image_size=64, patch_size=16, num_classes=10, dim=64, depth=0, heads=1, mlp_dim=1, dim_head=1)
    t2t_shell = oracle.make_config("t2t_vit", image_size=32, num_classes=10, dim=64, depth=0, heads=1, mlp_dim=1,
                                   t2t_layers=((3, 2), (3, 2)))
    identity = lambda x, training=True: x  # noqa: E731
    for cls, cfg, kw in ((vb.EfficientViT, shell, dict(image_size=64, patch_size=16)),
                         (vb.DistillableEfficientViT, shell, dict(image_size=64, patch_size=16)),
                         (vb.T2TViT, t2t_shell, dict(image_size=32, t2t_layers=((3, 2), (3, 2))))):
        out[f"{cls.__name__}:injected"] = ({cfg["kind"]: _names(oracle.weight_specs(cfg))},
                                           lambda seed, cls=cls, kw=kw: cls(**kw, num_classes=10, dim=64, transformer=identity, seed=seed),
                                           lambda seed, cfg=cfg: oracle.init_weights(cfg, seed))
    for mod in FAMILY_ORACLES:
        for name, kw in mod.SMALL.items():
            cfg = mod.make_config(**kw)
            out[f"{cfg['kind']}:{name}"] = ({cfg["kind"]: _names(mod.weight_specs(cfg))},
                                            lambda seed, cfg=cfg: vb.from_config(cfg, seed=seed),
                                            lambda seed, cfg=cfg, mod=mod: mod.init_weights(cfg, seed))
    # ATS-ViT's weights are ViT's, with to_out in every layer
    for name, c in ats_oracle.SMALL.items():
        K = c["max_tokens_per_depth"]
        cfg = _vit_cfg(c, len(K))
        out[f"ats_vit:{name}"] = ({"ats_vit": _names(oracle.weight_specs(cfg))},
                                  lambda seed, c=c, K=K: vb.ATSViT(image_size=c["image"], patch_size=c["patch"], num_classes=5,
                                                                   dim=c["dim"], depth=len(K), max_tokens_per_depth=K, heads=c["heads"],
                                                                   mlp_dim=c["mlp_dim"], dim_head=c["dim_head"], seed=seed),
                                  lambda seed, cfg=cfg: oracle.init_weights(cfg, seed))
    return out


ORACLE_CASES = _oracle_cases()


@pytest.mark.parametrize("seed", SEEDS)
@pytest.mark.parametrize("case", sorted(ORACLE_CASES))
def test_init_weights_match_the_oracle(monkeypatch, case, seed):
    specs, build, expected = ORACLE_CASES[case]
    engine = _SpecEngine(specs)
    monkeypatch.setattr(_lib, "load", lambda: engine)
    got, want = build(seed).get_weights_dict(), expected(seed)
    assert list(got) == list(want)
    for name, a in got.items():
        assert a.dtype == want[name].dtype and a.shape == want[name].shape and a.tobytes() == want[name].tobytes(), name


# ---- the classes without an initialising oracle: their weight lists restated from the engine's, and digests of the weights ----------
def _small_vit_specs(c):
    """ViT's list with SPT's LayerNorm over p^2 * 15 inputs before the patch Dense, to_out in every layer and a scalar temperature
    after each layer."""
    cfg = _vit_cfg(dict(c, patch=(c["patch"], c["patch"])), c["depth"])
    out = []
    for name, shape in _names(oracle.weight_specs(cfg)):
        if name == "patch.kernel":
            k = c["patch"] ** 2 * 15
            out += [("patch_norm.gamma", (k,)), ("patch_norm.beta", (k,)), ("patch.kernel", (k, c["dim"]))]
            continue
        out.append((name, shape))
        if name.endswith(".fc2.bias"):
            out.append((name[:-len("fc2.bias")] + "temperature", ()))
    return out


def _mim_specs(kind, c):
    """The encoder's weights but cls_token and the head, then the mask token, (MAE) enc_to_dec, the decoder and its positions,
    and to_pixels."""
    enc = _vit_cfg(c, c["depth"])
    out = [(n, s) for n, s in _names(oracle.weight_specs(enc)) if n != "cls_token" and not n.startswith("head")]
    dd = c["decoder_dim"] if kind == "mae" else c["dim"]
    pd = c["patch"][0] * c["patch"][1] * 3
    out.append(("mask_token", (dd,)))
    if kind == "mae":
        dec = {}
        if dd != c["dim"]:
            dec["enc_to_dec.kernel"], dec["enc_to_dec.bias"] = ((c["dim"], dd), None), ((dd,), None)
        for L in range(c["decoder_depth"]):
            _vit_layer(dec, f"decoder.layers.{L}.", dd, c["decoder_heads"], c["decoder_dim_head"], 4 * dd, kind="vit")
        out += _names(dec) + [("decoder_pos_emb.embeddings", (enc["num_patches"] + 1, dd))]
    return out + [("to_pixels.kernel", (dd, pd)), ("to_pixels.bias", (pd,))]


def _pinned_cases():
    out = {}
    for name, c in small_vit_oracle.SMALL.items():
        out[f"small_dataset_vit:{name}"] = (
            {"small_dataset_vit": _small_vit_specs(c)},
            lambda seed, c=c: vb.SmallDatasetViT(image_size=c["image"], patch_size=c["patch"], num_classes=5, dim=c["dim"],
                                                 depth=c["depth"], heads=c["heads"], mlp_dim=c["mlp_dim"], pool=c["pool"],
                                                 dim_head=c["dim_head"], seed=seed))
    for name, (kind, c) in mim_oracle.CASES.items():
        def build(seed, kind=kind, c=c):
            enc = vb.ViT(image_size=c["image"], patch_size=c["patch"], num_classes=5, dim=c["dim"], depth=c["depth"], heads=c["heads"],
                         mlp_dim=c["mlp_dim"], dim_head=c["dim_head"])
            if kind == "mae":
                return vb.MAE(image_size=c["image"][0], encoder=enc, decoder_dim=c["decoder_dim"], masking_ratio=c["ratio"],
                              decoder_depth=c["decoder_depth"], decoder_heads=c["decoder_heads"],
                              decoder_dim_head=c["decoder_dim_head"], seed=seed)
            return vb.SimMIM(image_size=c["image"][0], encoder=enc, masking_ratio=c["ratio"], seed=seed)
        out[f"{kind}:{name}"] = ({"vit": _names(oracle.weight_specs(_vit_cfg(c, c["depth"]))), kind: _mim_specs(kind, c)}, build)
    return out


PINNED_CASES = _pinned_cases()
# sha256 of (name, dtype, shape, bytes) of every weight, in order, as init_weights drew them when this test was written
PINNED = {
    "mae:mae_dense:0": "0c787630a5eba8ecf8bb7091", "mae:mae_dense:1": "0e95e873f6e05a201e5744f8",
    "mae:mae_identity:0": "90d1588930dfa2690b42ff26", "mae:mae_identity:1": "2b1a318ac26fd5d0439edd07",
    "mae:mae_no_to_out:0": "32ce2f2645c6e9ecd8c54b25", "mae:mae_no_to_out:1": "7840da37b42fb7efd4c3a516",
    "mae:mae_ratio29:0": "6c3bd66dbe6ecf0e60fd5718", "mae:mae_ratio29:1": "cf507fc85a96e43724d3c765",
    "mae:mae_readme:0": "7c8ed6954f93f0665b85e476", "mae:mae_readme:1": "cf96a0988b994524d5c02aee",
    "mae:mae_rect:0": "5590de76565d2796197be55a", "mae:mae_rect:1": "7090fd72635677f4f41f9d26",
    "mae:mae_small_image:0": "a244c0d8ae6433569e57be83", "mae:mae_small_image:1": "baddbb42eebaf98115683a08",
    "simmim:simmim_base:0": "14677eceb624c76e0e9e5b2c", "simmim:simmim_base:1": "9d281534b0be53d29ffabbef",
    "simmim:simmim_odd:0": "66fd79c0cf7354723cf6abea", "simmim:simmim_odd:1": "e207dbe1d0a459f6ddf8c8fa",
    "simmim:simmim_ratio29:0": "c65f11ee24127dbaef268ad1", "simmim:simmim_ratio29:1": "33aa072b3de7bb631efdf7c9",
    "simmim:simmim_readme:0": "9ffc46bf1a3d59f7bba53b46", "simmim:simmim_readme:1": "f18e811039142f5e0caab665",
    "simmim:simmim_rect:0": "c156b25e5fe3ac681c57b08a", "simmim:simmim_rect:1": "6ceaa966c17c0bb59fc8d48f",
    "simmim:simmim_small_image:0": "c65f11ee24127dbaef268ad1", "simmim:simmim_small_image:1": "33aa072b3de7bb631efdf7c9",
    "small_dataset_vit:rect_p4_dh80_mean:0": "0dad642dcade045b608399a6", "small_dataset_vit:rect_p4_dh80_mean:1": "8850d3d02620080dd4c59dd6",
    "small_dataset_vit:rect_p8_dh32_mean:0": "ae393de3465ba2f964857b72", "small_dataset_vit:rect_p8_dh32_mean:1": "e551fb972f7a09878c37039f",
    "small_dataset_vit:sq_p4_dh16:0": "595ad666122330e69b74c616", "small_dataset_vit:sq_p4_dh16:1": "f1d2890f30f43bc8fdccf49a",
    "small_dataset_vit:sq_p4_dh64:0": "3a61278730a1b535a8f1540d", "small_dataset_vit:sq_p4_dh64:1": "033c8cd6d5d70587377bcb5c",
    "small_dataset_vit:sq_p8_dh48:0": "d1f03a97c3154f1689df1fe3", "small_dataset_vit:sq_p8_dh48:1": "bf3ac9e4e57c1f081a111f28",
}


def _digest(weights):
    h = hashlib.sha256()
    for name, a in weights.items():
        h.update(f"{name} {a.dtype} {a.shape}\n".encode())
        h.update(a.tobytes())
    return h.hexdigest()[:24]


@pytest.mark.parametrize("seed", SEEDS)
@pytest.mark.parametrize("case", sorted(PINNED_CASES))
def test_init_weights_match_their_pinned_digest(monkeypatch, case, seed):
    specs, build = PINNED_CASES[case]
    engine = _SpecEngine(specs)
    monkeypatch.setattr(_lib, "load", lambda: engine)
    assert _digest(build(seed).get_weights_dict()) == PINNED[f"{case}:{seed}"]


def test_a_weight_without_an_initial_distribution_is_refused(monkeypatch):
    cfg = cases.cfg_of("vit_small")
    monkeypatch.setattr(_lib, "load", lambda: _SpecEngine({"vit": _names(oracle.weight_specs(cfg)) + [("layers.0.mystery", (2,))]}))
    with pytest.raises(AssertionError, match="layers.0.mystery"):
        vb.from_config(cfg, seed=0)


# ---- constructor refusals of the families with an extension config that set VbConfig's fields themselves ----------------------------
_LEVIT = dict(image_size=224, num_classes=10, dim=(64, 96, 128), depth=1, heads=(2, 3, 4), mlp_mult=2)
_NEST = dict(image_size=64, patch_size=4, num_classes=10, dim=32, heads=2, num_hierarchies=3, block_repeats=(1, 1, 1))
_FAMILIES = {"LeViT": (vb.LeViT, _LEVIT), "CvT": (vb.CvT, dict(num_classes=10)), "TwinsSVT": (vb.TwinsSVT, dict(num_classes=10)),
             "CrossFormer": (vb.CrossFormer, dict(num_classes=10)), "NesT": (vb.NesT, _NEST), "RegionViT": (vb.RegionViT, dict(num_classes=10))}
_PRECISION = "precision must be one of ['bf16', 'bfloat16', 'float32', 'fp32']"
# a non-integer num_classes is refused by ctypes when it is stored, after the precision check and before the extension config
_REFUSALS = [(dict(num_classes=2.5), TypeError, "'float' object cannot be interpreted as an integer"),
             (dict(num_classes=10.0), TypeError, "'float' object cannot be interpreted as an integer"),
             (dict(num_classes="10"), TypeError, "'str' object cannot be interpreted as an integer"),
             (dict(num_classes=None), TypeError, "'NoneType' object cannot be interpreted as an integer"),
             (dict(precision="fp64"), ValueError, _PRECISION),
             (dict(precision="fp64", num_classes=2.5), ValueError, _PRECISION)]


@pytest.mark.parametrize("i", range(len(_REFUSALS)))
@pytest.mark.parametrize("family", sorted(_FAMILIES))
def test_constructor_refusals(monkeypatch, family, i):
    cls, kw = _FAMILIES[family]
    extra, exc, message = _REFUSALS[i]
    monkeypatch.setattr(_lib, "load", lambda: _SpecEngine({}))
    with pytest.raises(exc) as e:
        cls(**{**kw, **extra})
    assert str(e.value) == message


@pytest.mark.parametrize("cls,kw", [(vb.LeViT, dict(_LEVIT, dim=(64.5, 96.5, 128.5))), (vb.NesT, dict(_NEST, dim=32.5))])
def test_bad_precision_is_refused_before_the_extension_config(monkeypatch, cls, kw):
    monkeypatch.setattr(_lib, "load", lambda: _SpecEngine({}))
    with pytest.raises(ValueError) as e:
        cls(**{**kw, "precision": "fp64"})
    assert str(e.value) == _PRECISION
