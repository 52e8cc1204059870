"""CPU: the nn.Module surface mirrors the reference (state_dict contract, factory, deepcopy, loud CPU failure)."""
import copy
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from latte_b200 import Latte, Latte_models
from latte_b200.models import get_models
from oracle import latte_oracle as O
from golden_sample import as_stored  # noqa: E402


def _small():
    return Latte(input_size=16, hidden_size=128, depth=2, num_heads=2, num_frames=8, num_classes=101, extras=2)


def test_state_dict_keys_match_reference_contract():
    cfg = O.make_config("Latte-tiny64/2", input_size=16, num_frames=8)
    net = _small()
    spec = dict(O.state_dict_spec(cfg))
    sd = net.state_dict()
    assert set(sd) == set(spec)
    for k, shape in spec.items():
        assert tuple(sd[k].shape) == tuple(shape), k
    # frozen tables, trainable everything else (SURVEY.md App. B)
    grads = {n: p.requires_grad for n, p in net.named_parameters()}
    assert not grads["pos_embed"] and not grads["temp_embed"]
    assert all(v for k, v in grads.items() if k not in ("pos_embed", "temp_embed"))


def test_reference_checkpoint_roundtrip():
    cfg = O.make_config("Latte-tiny64/2", input_size=16, num_frames=8)
    sd = O.make_weights(cfg, 3)
    net = _small()
    missing, unexpected = net.load_state_dict(sd, strict=True)
    assert not missing and not unexpected
    out = net.state_dict()
    for k in sd:
        assert torch.equal(out[k], sd[k]), k
    ema = copy.deepcopy(net)  # train.py:121
    assert torch.equal(ema.blocks[1].mlp.fc2.weight, net.blocks[1].mlp.fc2.weight)


def test_init_matches_reference_tables_and_zero_init(golden_dir):
    g = np.load(os.path.join(golden_dir, "subops_tiny72.npz"))
    net = Latte(input_size=16, hidden_size=576, depth=2, num_heads=8, num_frames=4, num_classes=5, extras=2)
    assert np.array_equal(as_stored(net.pos_embed.numpy(), g, "fresh_pos_embed"), g["fresh_pos_embed"])     # bit-exact sin-cos tables (latte.py:406-457)
    assert np.array_equal(net.temp_embed.numpy(), g["fresh_temp_embed"])
    assert float(net.final_layer.linear.weight.abs().max()) == 0.0          # adaLN-Zero (latte.py:286-295)
    assert all(float(b.adaLN_modulation[1].weight.abs().max()) == 0.0 for b in net.blocks)
    assert float(net.blocks[0].attn.qkv.bias.abs().max()) == 0.0


def test_size_table_and_factory():
    assert set(Latte_models) == {f"Latte-{s}/{p}" for s in ("XL", "L", "B", "S") for p in (2, 4, 8)}
    args = SimpleNamespace(model="Latte-S/2", latent_size=32, num_classes=101, num_frames=16, learn_sigma=True, extras=2)
    net = get_models(args)
    assert isinstance(net, Latte) and net.hidden_size == 384 and net.depth == 12 and net.num_heads == 6
    assert net.in_channels == 4 and net.out_channels == 8 and net.learn_sigma and net.num_frames == 16
    assert sum(p.numel() for p in net.parameters()) == 32_624_288  # reference S/2 parameter count (SURVEY.md App. D)
    with pytest.raises(NotImplementedError):
        get_models(SimpleNamespace(model="LatteIMG-XL/2"))


def test_unpatchify_matches_reference(golden_dir):
    g = np.load(os.path.join(golden_dir, "subops_tiny72.npz"))
    net = Latte(input_size=16, hidden_size=128, depth=2, num_heads=2, num_frames=4, num_classes=5, extras=2)
    x = torch.arange(2 * 64 * 32, dtype=torch.float32).reshape(2, 64, 32)
    assert np.array_equal(net.unpatchify(x).numpy(), g["unpatchify"])


def test_no_cpu_fallback():
    net = _small().eval()
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        net(torch.randn(2, 8, 4, 16, 16), torch.tensor([1, 2]), y=torch.tensor([0, 1]))
    from latte_b200 import ops
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.linear(torch.zeros(128, 64, dtype=torch.float16), torch.zeros(128, 64, dtype=torch.float16))


def test_unsupported_variants_fail_loudly():
    with pytest.raises(NotImplementedError):
        Latte(extras=78)
    with pytest.raises(NotImplementedError):
        Latte(attention_mode="flash")


def test_product_never_imports_oracle():
    """The product package must not import or call oracle/ (parity claims are void otherwise)."""
    import re
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    pat = re.compile(r"^\s*(import|from)\s+\.*oracle\b|\boracle\.[a-z_]+\(", re.M)
    for dp, _, files in os.walk(os.path.join(root, "latte_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                text = open(os.path.join(dp, f)).read()
                assert not pat.search(text), f


def test_dropin_packages_import_through_symlinks(tmp_path):
    """INTEGRATION.md section 3: `models` and `diffusion` put ahead of the reference's on sys.path as symlinks to
    latte_b200/models and latte_b200/diffusion must import as TOP-LEVEL packages (ADVICE r01: relative imports broke it)."""
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    os.symlink(os.path.join(root, "latte_b200", "models"), tmp_path / "models")
    os.symlink(os.path.join(root, "latte_b200", "diffusion"), tmp_path / "diffusion")
    code = ("import models, diffusion; from types import SimpleNamespace as N; "
            "m = models.get_models(N(model='Latte-S/2', latent_size=32, num_classes=101, num_frames=16, learn_sigma=True, extras=2)); "
            "d = diffusion.create_diffusion('250'); print(type(m).__name__, d.num_timesteps)")
    env = dict(os.environ, PYTHONPATH=f"{tmp_path}{os.pathsep}{root}", LATTE_B200_NO_BUILD="1")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, cwd=str(tmp_path))
    assert r.returncode == 0, r.stderr
    assert r.stdout.split() == ["Latte", "250"]


def test_device_caches_are_not_pickled():
    """copy.deepcopy (EMA, train.py:95-97) and pickle must work after the packing cache holds ctypes pointer structs."""
    import copy
    import pickle
    from latte_b200 import Latte, _lib
    from latte_b200.diffusion import create_diffusion
    net = Latte(input_size=16, hidden_size=128, depth=2, num_heads=2, num_frames=4, num_classes=5, extras=2)
    net._packed = (_lib.LatteShape(), _lib.LatteWeights(), {}, None)      # what a forward leaves behind
    net._graphs = {"k": object()}
    twin = copy.deepcopy(net)
    assert twin._packed is None and twin._graphs is None
    assert all(torch.equal(a, b) for a, b in zip(net.state_dict().values(), twin.state_dict().values()))
    pickle.loads(pickle.dumps(net))
    d = create_diffusion("8")
    d._dev["x"] = _lib.SamplerTables()
    assert copy.deepcopy(d)._dev == {}


def test_mask_text_embeddings_matches_pipeline_semantics():
    """pipeline_latte.py:118-124: one prompt is trimmed to its kept tokens, a batch is zero-masked and keeps its length."""
    from latte_b200.t5 import mask_text_embeddings
    emb = torch.arange(2 * 1 * 6 * 4, dtype=torch.float32).reshape(2, 1, 6, 4) + 1
    mask = torch.tensor([[1, 1, 1, 0, 0, 0], [1, 1, 1, 1, 1, 0]])
    one, keep = mask_text_embeddings(emb[:1], mask[:1])
    assert keep == 3 and one.shape == (1, 1, 3, 4) and torch.equal(one, emb[:1, :, :3])
    both, length = mask_text_embeddings(emb, mask)
    assert length == 6 and torch.equal(both[0, 0, 3:], torch.zeros(3, 4)) and torch.equal(both[1, 0, :5], emb[1, 0, :5])


def test_utils_surface_and_no_cpu_fallback():
    """latte_b200.utils mirrors the reference's utils.clip_grad_norm_ / update_ema / requires_grad (train.py:36-38)."""
    import inspect
    from latte_b200 import utils as U
    assert list(inspect.signature(U.clip_grad_norm_).parameters) == ["parameters", "max_norm", "norm_type", "error_if_nonfinite", "clip_grad"]
    assert list(inspect.signature(U.update_ema).parameters) == ["ema_model", "model", "decay"]
    p = torch.nn.Parameter(torch.ones(8))
    p.grad = torch.ones(8)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        U.clip_grad_norm_([p], 1.0)
    with pytest.raises(NotImplementedError):
        U.clip_grad_norm_([p], 1.0, norm_type=float("inf"))
    assert U.clip_grad_norm_([torch.nn.Parameter(torch.ones(2))], 1.0).item() == 0.0      # no gradients at all
    net = torch.nn.Linear(2, 2)
    U.requires_grad(net, False)
    assert not any(q.requires_grad for q in net.parameters())
