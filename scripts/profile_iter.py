"""One-wave slice of the c2 workload for ncu: prologue + a few CEM-iteration launches."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from tdmpc2_b200.config import workload
from tdmpc2_b200.synth import synth_state_dict
from tdmpc2_b200.planner import Planner, draw_noise

wl = sys.argv[1] if len(sys.argv) > 1 else "c2"
E = int(sys.argv[2]) if len(sys.argv) > 2 else 37
iters = int(sys.argv[3]) if len(sys.argv) > 3 else 3
cfg = workload(wl, num_envs=E)
pl = Planner(cfg, E, "cuda:0", engine=os.environ.get("TDMPC2_ENGINE"))     # None: the default engine (tcgen05)
pl.pack(synth_state_dict(cfg, seed=1))
dev = torch.device("cuda:0")
n = draw_noise(cfg, E, dev, reference_order=False)
NSM = torch.cuda.get_device_properties(0).multi_processor_count
obs = torch.randn(E, cfg.obs_shape["state"][0], device=dev)
task = (torch.arange(E) % len(cfg.tasks)).to(torch.int32).to(dev) if cfg.multitask else None
pl.prologue(obs, task, torch.ones(E, dtype=torch.uint8, device=dev), torch.zeros(E, cfg.horizon, cfg.action_dim, device=dev), n.prior)
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
for i in range(iters):
    a = (n.r[i % cfg.iterations], n.pi[i % cfg.iterations], n.qidx[i % cfg.iterations])
    e0.record(); pl.iterate(*a); e1.record(); torch.cuda.synchronize()
    print(f"iter {i}: {e0.elapsed_time(e1):.3f} ms (E={E}, tiles={E * ((cfg.num_samples + 127) // 128)})")

if os.environ.get("TDMPC2_PHASE_PROF"):
    buf = torch.zeros(NSM * 4 * 12 + 32 * 16, dtype=torch.int64, device=dev)
    pl.lib.tdmpc2_planner_set_profile(pl.h, buf.data_ptr())
    a = (n.r[0], n.pi[0], n.qidx[0])
    pl.iterate(*a); torch.cuda.synchronize()
    pl.lib.tdmpc2_planner_set_profile(pl.h, None)
    b = buf[:NSM * 4 * 12].view(NSM, 4, 12).double().cpu()
    tr = buf[NSM * 4 * 12:].view(32, 16).cpu()
    names = ["producer", "mma", "epilogue", "idle"]
    cols = ["bar_wait", "in_layers", "facc_wait", "publish", "setup", "kernel", "actions", "refit", "decode"]
    m = b.mean(0)
    print("refit max over CTAs: %.1fk  kernel max: %.1fk min: %.1fk" % (b[:, 3, 7].max() / 1e3, b[:, 3, 5].max() / 1e3, b[:, 3, 5].min() / 1e3))
    for r in range(4):
        print(names[r].ljust(10), "  ".join(f"{cols[k]}={m[r, k] / 1e3:9.1f}k" for k in range(9)))

    if os.environ.get("TDMPC2_TRACE") == "pp":
        ev = ["start", "gA0", "gA1", "gB0", "gB1", "accA", "eA", "eAend", "accB", "eB", "eBend"]
        t00 = int(tr[0, 0])
        for st in range(27):
            t0 = int(tr[st, 0])
            print(f"step {st:2d} @{(t0 - t00) / 1e3:8.1f}k  " + " ".join(f"{ev[k]}={(int(tr[st, k]) - t0) / 1e3:6.1f}" for k in range(1, 11) if int(tr[st, k]) > 0))
    elif os.environ.get("TDMPC2_TRACE"):
        ev = ["start", "tma0", "mma0", "mmaL", "e0acc", "e0p1", "e0bar", "e0p2", "e0bw", "end", "e3acc", "e3p2"]
        t00 = int(tr[0, 0])
        for st in range(27):
            t0 = int(tr[st, 0])
            print(f"step {st:2d} @{(t0 - t00) / 1e3:8.1f}k  " + " ".join(f"{ev[k]}={(int(tr[st, k]) - t0) / 1e3:6.1f}" for k in range(1, 12) if int(tr[st, k]) > 0))
