"""Debug: which entries of d(output.bias) disagree with the oracle for the R101-L1-H2048 architecture (B=2)."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import torch
from oracle import virtex_oracle as O
from tests.helpers import build_model, to_cuda
from tests.test_gpu_parity import rel, cos

for kw in (dict(backbone="resnet101", hidden=2048, heads=32, ffn=8192), dict(hidden=2048, heads=32, ffn=8192),
           dict(backbone="resnet101")):
    spec = O.Spec(**kw)
    state = O.synth_state(spec, 12, bn3_gain=0.25)
    model = build_model(spec, state)
    model.train()
    batch = O.synth_batch(2, seed=8, ragged=False)
    out = model(to_cuda(batch))
    ref, grads, _ = O.loss_and_grads(state, batch, spec)
    out["loss"].backward()
    torch.cuda.synchronize()
    eng = model.engine
    g = eng.G("textual.output.bias").float().cpu()
    gr = grads["textual.output.bias"]
    print(kw, "loss", out["loss"].item(), ref["loss"].item(), "bias rel", rel(g, gr), "cos", cos(g, gr))
    # recompute from the dlogits the engine left behind
    s = sum(r["logits"].float().sum(0) for r in eng._recs).cpu()
    print("  torch colsum of dlogits vs engine:", rel(g, s), " vs oracle:", rel(s, gr))
    d = (g - gr).abs()
    bad = (d > 0.05 * gr.abs().max()).nonzero().flatten()
    print("  n bad", bad.numel(), "first", bad[:10].tolist(), "last", bad[-10:].tolist())
    for r in eng._recs:
        print("   dir", r["direction"], "dlogits absmax", r["logits"].abs().max().item(), "nan", torch.isnan(r["logits"].float()).any().item())
    # per-direction oracle bias grads are not available; compare fwd logits instead
    with torch.no_grad():
        o = O.model_forward(state, batch, spec, training=True, return_logits=True)
    eng.forward(batch["image"].cuda(), batch["caption_tokens"].cuda(), batch["noitpac_tokens"].cuda(),
                batch["caption_lengths"].cuda(), training=True, with_grad=False)
    lg = eng._recs[0]["logits"].float().view(2, 30, -1).cpu()
    print("  fwd logits max abs err", (lg - o["logits"]).abs().max().item(), "bwd",
          (eng._recs[1]["logits"].float().view(2, 30, -1).cpu() - o["backward_logits"]).abs().max().item())
    del model, eng
    torch.cuda.empty_cache()
