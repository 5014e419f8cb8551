"""CAM / EdgeDisplacement errors against the reference goldens for a conv mode (development aid).
    python tools/net_err.py [mode=2]"""
import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from irn_b200 import preprocess, synth
from irn_b200.cam import CAM
from irn_b200.irn import EdgeDisplacement

mode = int(sys.argv[1]) if len(sys.argv) > 1 else 2
dev = torch.device("cuda:0")
G = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
g = np.load(os.path.join(G, "steps512.npz"))
cam, irn = CAM(), EdgeDisplacement()
cam.load_state_dict(synth.cam_state_dict(), strict=True)
irn.load_state_dict(synth.irn_state_dict(), strict=False)
cam.cuda(dev), irn.cuda(dev)
cam.set_conv_mode(mode), irn.set_conv_mode(mode)
x = torch.from_numpy(synth.image(int(g["seed"]), 512, 512)[None]).to(dev)
pyr = preprocess.msf_batch(x, (1.0, 0.5, 1.5, 2.0))
out = {"mode": mode, "env": {k: v for k, v in os.environ.items() if k.startswith("IRN_F16")}}
for p in pyr:
    ref = g["camscale_%d" % p.shape[-1]]
    y = cam(p).cpu().numpy()
    out["cam_%d" % p.shape[-1]] = float(np.abs(y - ref).max() / ref.max())
e, d = irn(pyr[0])
out["edge"] = float(np.abs(e.cpu().numpy() - g["edge"]).max())
out["dp"] = float(np.abs(d.cpu().numpy() - g["dp"]).max())
gc = np.load(os.path.join(G, "cam_forward.npz"))
for i in range(3):
    y = cam(torch.from_numpy(gc["x%d" % i]).to(dev)).cpu().numpy()
    out["cam_small%d" % i] = float(np.abs(y - gc["y%d" % i]).max() / gc["y%d" % i].max())
gi = np.load(os.path.join(G, "irn_forward.npz"))
for i in range(2):
    e, d = irn(torch.from_numpy(gi["x%d" % i]).to(dev))
    out["edge_small%d" % i] = float(np.abs(e.cpu().numpy() - gi["edge%d" % i]).max())
    out["dp_small%d" % i] = float(np.abs(d.cpu().numpy() - gi["dp%d" % i]).max())
print(json.dumps(out), flush=True)
