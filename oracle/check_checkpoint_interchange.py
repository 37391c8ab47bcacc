"""One-off cross-check (TEST INFRASTRUCTURE, needs a reference checkout in $VIRTEX_REFERENCE_ROOT): checkpoints written by the UNMODIFIED reference
(`virtex.utils.checkpointing.CheckpointManager` around its model + Lookahead(SGD) + LinearWarmupCosineAnnealingLR) load
into virtex_b200's model and fused-optimiser state views, and checkpoints written by virtex_b200 load back into the
reference objects (strict key match, momentum buffers bit-equal, schedule continues at the same learning rate).

    python oracle/check_checkpoint_interchange.py        # prints three "OK" lines

The reference runs in subprocesses because its package name (`virtex`) is also this repo's alias package.
"""
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OVERRIDES = ["MODEL.TEXTUAL.NAME", "transdec_postnorm::L1_H128_A2_F256", "OPTIM.CNN_LR", 0.1, "OPTIM.LR", 0.001,
             "OPTIM.WARMUP_STEPS", 4, "OPTIM.NUM_ITERATIONS", 20]

REF_SIDE = r'''
import sys
mode, work, root = sys.argv[1], sys.argv[2], sys.argv[3]
sys.path.insert(0, root)
from oracle import ref_shim
ref_shim.install()
sys.path.insert(0, ref_shim.REFERENCE_ROOT)
for k in [k for k in sys.modules if k == "virtex" or k.startswith("virtex.")]:
    del sys.modules[k]
import torch
from virtex.config import Config
from virtex.factories import PretrainingModelFactory, OptimizerFactory, LRSchedulerFactory
from virtex.utils.checkpointing import CheckpointManager
c = Config(ref_shim.REFERENCE_ROOT + "/configs/_base_bicaptioning_R_50_L1_H1024.yaml", %r)
torch.manual_seed(1)
m = PretrainingModelFactory.from_config(c)
opt = OptimizerFactory.from_config(c, m.named_parameters())
sch = LRSchedulerFactory.from_config(c, opt)
mgr = CheckpointManager(work + "/ref", model=m, optimizer=opt, scheduler=sch)
if mode == "write":
    import os
    os.makedirs(work + "/ref", exist_ok=True)
    for it in range(3):
        for p in m.parameters():
            p.grad = torch.randn_like(p) * 0.01
        opt.step(); sch.step()
    mgr.step(3)
    print("OK reference wrote checkpoint_3.pth")
else:
    it = mgr.load(work + "/ours/checkpoint_7.pth")
    ck = torch.load(work + "/ours/checkpoint_7.pth", weights_only=False)
    sd = opt.state_dict()
    assert it == 7 and sch.last_epoch == 7 and len(sd["state"]) == len(sd["param_groups"])
    assert all(torch.equal(sd["state"][i]["momentum_buffer"], ck["optimizer"]["state"][i]["momentum_buffer"]) for i in sd["state"])
    assert all(torch.equal(v, ck["model"][k]) for k, v in m.state_dict().items())
    opt.step(); sch.step()
    print("OK reference loaded virtex_b200's checkpoint_7.pth and kept training, lr", sch.get_last_lr()[0])
''' % (OVERRIDES,)


def ours(work):
    import torch
    sys.path.insert(0, ROOT)
    from tests.test_host_cpu import _fake_trainer, _tiny_config
    from virtex_b200.checkpointing import CheckpointManager, FusedOptimizerState, FusedSchedulerState
    from virtex_b200.factories import PretrainingModelFactory
    cfg = _tiny_config()
    model = PretrainingModelFactory.from_config(cfg)
    tr = _fake_trainer(model, cfg)
    mgr = CheckpointManager(work + "/ours", model=model, optimizer=FusedOptimizerState(tr),
                            scheduler=FusedSchedulerState(tr))
    it = mgr.load(work + "/ref/checkpoint_3.pth")
    ck = torch.load(work + "/ref/checkpoint_3.pth", weights_only=False)
    assert it == 3 and not mgr.not_loaded and not mgr.not_found and tr.iteration == 3 and tr.momentum_ready
    assert all(torch.equal(tr.arena.view(tr.mom, n), ck["optimizer"]["state"][i]["momentum_buffer"])
               for i, n in enumerate(tr.arena.names))
    assert len(ck["model"]) == 370 and all(torch.equal(v, ck["model"][k]) for k, v in model.state_dict().items())
    tr.iteration = 7
    mgr.step(7)
    print("OK virtex_b200 loaded the reference's checkpoint_3.pth (370 model keys, 202 momentum buffers) and wrote "
          "checkpoint_7.pth")


if __name__ == "__main__":
    with tempfile.TemporaryDirectory() as work:
        script = os.path.join(work, "ref_side.py")
        with open(script, "w") as f:
            f.write(REF_SIDE)
        subprocess.run([sys.executable, script, "write", work, ROOT], check=True, cwd=work)
        ours(work)
        subprocess.run([sys.executable, script, "read", work, ROOT], check=True, cwd=work)
