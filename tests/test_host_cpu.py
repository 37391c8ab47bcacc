"""CPU-side checks: module tree / state_dict compatibility, C-ABI library loads and exports every declared symbol."""
import ctypes
import os
import re

import pytest
import torch

from oracle import virtex_oracle as O
from tests.helpers import virtex_model

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_state_dict_matches_reference_key_set():
    spec = O.Spec()
    model = virtex_model(spec, dropout=0.1)
    ref_sd = O.to_reference_state_dict(O.synth_state(spec, 0), spec)
    sd = model.state_dict()
    assert set(sd) == set(ref_sd)
    assert len(sd) == 370
    for k, v in ref_sd.items():
        assert tuple(sd[k].shape) == tuple(v.shape), k
    assert sum(p.numel() for p in model.parameters()) == 69_482_320
    assert len(list(model.parameters())) == 202
    model.load_state_dict(ref_sd, strict=True)


def test_weight_sharing_and_init():
    spec = O.Spec(hidden=128, layers=2, heads=2, ffn=256)
    m = virtex_model(spec, dropout=0.1)
    assert m.backward_textual.embedding is m.textual.embedding
    assert m.backward_textual.visual_projection is m.textual.visual_projection
    assert m.backward_textual.output is m.textual.output
    assert m.textual.output.weight is m.textual.embedding.words.weight
    assert m.backward_textual.transformer is not m.textual.transformer
    assert torch.all(m.textual.embedding.words.weight[0] == 0)
    # zero_init_residual
    assert torch.all(m.visual.cnn.layer1[0].bn3.weight == 0)
    assert abs(m.textual.transformer.layers[0].linear1.weight.std().item() - 0.02) < 2e-3


def test_no_cpu_fallback():
    spec = O.Spec(hidden=128, layers=1, heads=2, ffn=256)
    m = virtex_model(spec, dropout=0.1)
    batch = O.synth_batch(2, 0)
    with pytest.raises(RuntimeError, match="no CPU path"):
        m(batch)


def test_library_exports_every_declared_symbol():
    from virtex_b200 import lib as L, ops
    header = open(os.path.join(ROOT, "include", "virtex_b200.h")).read()
    declared = set(re.findall(r"\b(vtx_[a-z0-9_]+)\s*\(", header))
    so = ctypes.CDLL(L.LIB_PATH)
    for name in declared:
        assert hasattr(so, name), f"{name} declared in include/virtex_b200.h but not exported"
    assert declared == set(ops.exported_symbols())
    assert so.vtx_version() >= 100


def test_ctypes_gemm_struct_mirrors_the_header_field_for_field():
    """`virtex_b200.lib.VtxGemm` (what every GEMM call marshals) against `typedef struct VtxGemm` of
    include/virtex_b200.h: same field names in the same order, C types of the same width, and the size the built
    library reports -- so an edit of either side that forgets the other fails here, not as a corrupted launch."""
    from virtex_b200 import lib as L
    header = open(os.path.join(ROOT, "include", "virtex_b200.h")).read()
    body = header[header.index("typedef struct VtxGemm {"):header.index("} VtxGemm;")]
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S).split("{", 1)[1]
    fields = []
    for decl in body.split(";"):
        decl = decl.strip()
        if not decl:
            continue
        ctype, names = decl.rsplit(" ", 1)[0], decl
        # "int64_t lda, ldb, ldd, ldr" / "const void* A" / "float* stats"
        m = re.match(r"(const\s+)?(\w+)\s*(\*?)\s*(.*)", decl)
        base, ptr, rest = m.group(2), m.group(3), m.group(4)
        for name in rest.split(","):
            name = name.strip()
            is_ptr = bool(ptr) or name.startswith("*")
            fields.append((name.lstrip("* "), "ptr" if is_ptr else base))
    width = {"ptr": 8, "int64_t": 8, "int32_t": 4, "float": 4}
    mirror = [(n, ctypes.sizeof(t)) for n, t in L.VtxGemm._fields_]
    assert [n for n, _ in fields] == [n for n, _ in mirror]
    assert [width[t] for _, t in fields] == [w for _, w in mirror]
    assert ctypes.CDLL(L.LIB_PATH).vtx_sizeof_gemm() == ctypes.sizeof(L.VtxGemm)


def test_virtex_alias_package_and_hubconf():
    """`import virtex.*` paths of the reference resolve to this implementation; hubconf exposes resnet50()."""
    import importlib
    import sys
    for m in [k for k in sys.modules if k == "virtex" or k.startswith("virtex.")]:
        del sys.modules[m]
    from virtex.config import Config
    from virtex.factories import PretrainingModelFactory, TextualHeadFactory
    from virtex.models import VirTexModel
    from virtex.modules.textual_heads import TransformerDecoderTextualHead
    import virtex_b200.models as vm
    assert VirTexModel is vm.VirTexModel
    assert set(TextualHeadFactory.PRODUCTS) == {"transdec_prenorm", "transdec_postnorm"}
    assert {"virtex", "bicaptioning", "captioning"} <= set(PretrainingModelFactory.PRODUCTS)
    with pytest.raises(KeyError):
        PretrainingModelFactory.create("does_not_exist")
    with pytest.raises(ValueError):
        PretrainingModelFactory()
    cfg = Config(None, ["MODEL.TEXTUAL.NAME", "transdec_prenorm::L2_H128_A2_F256"])
    head = TextualHeadFactory.from_config(cfg)
    assert isinstance(head, TransformerDecoderTextualHead) and head.norm_first and head.num_layers == 2
    with pytest.raises(KeyError):
        Config(None, ["OPTIM.DOES_NOT_EXIST", 1])
    with pytest.raises(ValueError):
        Config(None, ["OPTIM.BATCH_SIZE", "not-an-int"])
    hub = importlib.import_module("hubconf")
    m = hub.resnet50()
    sd = m.state_dict()
    assert "conv1.weight" in sd and "layer4.2.bn3.running_var" in sd and not any(k.startswith("fc.") for k in sd)
    assert len(sd) == 318
    assert m.layer3[0].conv1.weight.shape == (256, 512, 1, 1)


def test_config_yaml_inheritance_dump_and_freeze(tmp_path):
    from virtex_b200.config import Config
    c = Config("depth_ablations/bicaptioning_R_50_L4_H1024.yaml", ["OPTIM.BATCH_SIZE", 2048, "OPTIM.LR", "0.002"])
    assert c.MODEL.TEXTUAL.NAME == "transdec_postnorm::L4_H1024_A16_F4096"   # delta file
    assert c.MODEL.VISUAL.NAME == "torchvision::resnet50" and c.OPTIM.CNN_LR == 0.2  # inherited through _BASE_
    assert c.OPTIM.BATCH_SIZE == 2048 and c.OPTIM.LR == 0.002                  # override list, literal-evaluated
    with pytest.raises(AttributeError):
        c.OPTIM.LR = 1.0
    out = tmp_path / "dump.yaml"
    c.dump(str(out))
    c2 = Config(str(out))
    assert str(c2) == str(c)
    assert "BATCH_SIZE: 2048" in str(c)


def test_lr_schedules_and_lookahead_match_oracle_formulas():
    import torch
    from virtex_b200 import optim as vo
    cfg = O.OptimCfg(warmup_steps=5, num_iterations=40)
    fn = vo.lr_multiplier_fn("cosine", 40, 5)
    for s in range(0, 40):
        assert abs(fn(s) - O.lr_multiplier(s, cfg)) < 1e-12
    assert vo.lr_multiplier_fn("linear", 40, 5)(40) == 0.0 and vo.lr_multiplier_fn("none", 40, 5)(20) == 1.0
    assert abs(vo.lr_multiplier_fn("multistep", 40, 5, [10, 20], 0.1)(25) - 0.01) < 1e-12
    # Lookahead wrapper: k fast steps then interpolation towards the slow weights
    p = torch.nn.Parameter(torch.ones(4))
    opt = vo.Lookahead(torch.optim.SGD([p], lr=0.5), k=2, alpha=0.5)
    sched = vo.LinearWarmupCosineAnnealingLR(opt, total_steps=40, warmup_steps=5)
    assert opt.param_groups[0]["lr"] == 0.0     # lambda(0) = 0: the first step runs at lr 0 (SURVEY section 8a)
    for g in opt.param_groups:
        g["lr"] = 0.5
    p.grad = torch.ones(4); opt.step()           # fast: 1 - 0.5 = 0.5
    assert torch.allclose(p.data, torch.full((4,), 0.5))
    p.grad = torch.ones(4); opt.step()           # fast: 0.0 -> lookahead: 0.5*0.0 + 0.5*1.0 = 0.5
    assert torch.allclose(p.data, torch.full((4,), 0.5))
    assert torch.allclose(opt.state[p]["slow_params"], torch.full((4,), 0.5))
    assert sched is not None


# ------------------------------------------------------------------------------------------ checkpoint interchange
def _tiny_config():
    from virtex_b200.config import Config
    return Config(None, ["MODEL.TEXTUAL.NAME", "transdec_postnorm::L1_H128_A2_F256", "OPTIM.CNN_LR", 0.1,
                         "OPTIM.LR", 0.001, "OPTIM.WARMUP_STEPS", 4, "OPTIM.NUM_ITERATIONS", 20])


def _fake_trainer(model, config, device="cpu"):
    """The host-side state of `Trainer` without a GPU: real Arena (on the CPU) + the fields the state views read."""
    import types
    from virtex_b200.engine import Arena
    from virtex_b200.optim import lr_multiplier_fn
    named = [(n, p) for n, p in model.named_parameters()]
    t = types.SimpleNamespace()
    t.config = config
    t.arena = Arena(named, device)
    t.mom = torch.zeros_like(t.arena.params)
    t.slow = t.arena.params.clone()
    t.momentum = float(config.OPTIM.SGD_MOMENTUM)
    O = config.OPTIM
    t.lr_fn = lr_multiplier_fn(O.LR_DECAY_NAME, O.NUM_ITERATIONS, O.WARMUP_STEPS, O.LR_STEPS, O.LR_GAMMA)
    t.iteration, t._k_counter, t.momentum_ready = 0, 3, False

    def reset_lookahead():
        t._k_counter = 0
        t.slow.copy_(t.arena.params)
    t.reset_lookahead = reset_lookahead
    return t


def test_checkpoint_interchange_with_torch_optimizer_and_scheduler(tmp_path):
    """A checkpoint written by the reference's recipe (torch SGD in Lookahead + LambdaLR, one group per parameter) loads
    into the fused-tail state views, and what the views write loads back into the torch objects unchanged."""
    from virtex_b200.checkpointing import CheckpointManager, FusedOptimizerState, FusedSchedulerState
    from virtex_b200.factories import LRSchedulerFactory, OptimizerFactory, PretrainingModelFactory
    cfg = _tiny_config()
    torch.manual_seed(0)
    model = PretrainingModelFactory.from_config(cfg)
    opt = OptimizerFactory.from_config(cfg, model.named_parameters())
    sch = LRSchedulerFactory.from_config(cfg, opt)
    for it in range(3):  # momentum buffers + an advanced schedule
        for p in model.parameters():
            p.grad = torch.randn_like(p) * 0.01
        opt.step()
        sch.step()
    CheckpointManager(str(tmp_path / "ref"), model=model, optimizer=opt, scheduler=sch).step(3)

    # ---- "reference" checkpoint -> fused-tail views
    model2 = PretrainingModelFactory.from_config(cfg)
    tr = _fake_trainer(model2, cfg)
    mgr = CheckpointManager(str(tmp_path / "ours"), keep_recent=2, model=model2, optimizer=FusedOptimizerState(tr),
                            scheduler=FusedSchedulerState(tr))
    assert mgr.load(str(tmp_path / "ref" / "checkpoint_3.pth")) == 3
    assert mgr.not_loaded == [] and mgr.not_found == []
    assert tr.iteration == 3 and tr.momentum_ready and tr._k_counter == 0
    sd = opt.state_dict()
    names = tr.arena.names
    assert len(sd["param_groups"]) == len(names) == len(list(model.named_parameters()))
    for i, n in enumerate(names):
        assert torch.equal(tr.arena.view(tr.mom, n), sd["state"][i]["momentum_buffer"]), n
        assert torch.equal(tr.arena.p(n), dict(model.named_parameters())[n]), n
    assert torch.equal(tr.slow, tr.arena.params)  # Lookahead restarts from the loaded weights (as in the reference)

    # ---- fused-tail views -> file -> fresh torch optimizer / scheduler
    for it in (3, 4, 5):
        mgr.step(it, metric=1.0 / it)
    assert sorted(p.name for p in (tmp_path / "ours").iterdir()) == ["checkpoint_4.pth", "checkpoint_5.pth",
                                                                      "checkpoint_best.pth"]
    ck = torch.load(tmp_path / "ours" / "checkpoint_best.pth", weights_only=False)
    assert ck["iteration"] == 3  # 1/3 is the best ("higher is better") metric
    model3 = PretrainingModelFactory.from_config(cfg)
    opt3 = OptimizerFactory.from_config(cfg, model3.named_parameters())
    sch3 = LRSchedulerFactory.from_config(cfg, opt3)
    mgr3 = CheckpointManager(str(tmp_path / "x"), model=model3, optimizer=opt3, scheduler=sch3)
    assert mgr3.load(str(tmp_path / "ours" / "checkpoint_5.pth")) == 5
    sd3 = opt3.state_dict()
    for g, g3 in zip(sd["param_groups"], sd3["param_groups"]):
        for k in ("lr", "weight_decay", "momentum", "initial_lr", "params", "nesterov", "dampening"):
            assert g[k] == pytest.approx(g3[k], rel=1e-12, abs=0), k
    for i in range(len(names)):
        assert torch.equal(sd["state"][i]["momentum_buffer"], sd3["state"][i]["momentum_buffer"])
    assert sch3.last_epoch == 3 and sch3.get_last_lr() == pytest.approx(sch.get_last_lr())
    # and the schedule keeps going where it stopped
    opt3.step(); sch3.step(); opt.step(); sch.step()
    assert sch3.get_last_lr() == pytest.approx(sch.get_last_lr())


def test_fused_optimizer_state_is_empty_before_the_first_step_and_skips_frozen_parameters():
    from virtex_b200.checkpointing import FusedOptimizerState
    from virtex_b200.factories import PretrainingModelFactory
    cfg = _tiny_config()
    model = PretrainingModelFactory.from_config(cfg)
    for p in model.visual.parameters():
        p.requires_grad = False
    tr = _fake_trainer(model, cfg)
    view = FusedOptimizerState(tr)
    sd = view.state_dict()
    assert sd["state"] == {} and len(sd["param_groups"]) == len(tr.arena.names)
    assert all(g["lr"] == 0.0 for g in sd["param_groups"])  # LambdaLR: the first step runs at lambda(0) = 0
    tr.momentum_ready, tr.iteration = True, 2
    sd = view.state_dict()
    frozen = [i for i, n in enumerate(tr.arena.names) if n.startswith("visual.")]
    assert frozen and all(i not in sd["state"] for i in frozen)
    assert sd["param_groups"][frozen[0]]["lr"] == pytest.approx(0.1 * 2 / 4)
    with pytest.raises(ValueError):
        view.load_state_dict({"state": {}, "param_groups": sd["param_groups"][:-1]})
