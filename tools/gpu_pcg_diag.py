import os, sys
R = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, R); sys.path.insert(0, os.path.join(R, "tests"))
import numpy as np
from oracle_util import load_oracle
from lfr_b200 import build_problem, synth
from lfr_b200.capi import Plan, load_b200
lib = load_b200(); orc = load_oracle()
p = build_problem(synth.generate(sys.argv[1] if len(sys.argv) > 1 else "ring200"))
plan = Plan(lib, p, lib.default_options(debug_flags=0x10))  # LFR_DBG_PROFILE
plan.solve()
pos_g, st_g = plan.download()
rec, _ = plan.profile()
cta = rec["tier"] == 4
cg = rec["counter"].astype(np.int64)  # CG iterations on the CTA tier
pos_o, st_o = orc.solve(p, orc.default_options(n_threads=8))
sizes = np.diff(p.comp_ptr.astype(np.int64))
bad = np.nonzero(st_g["iterations"] != st_o["iterations"])[0]
print("mismatching comps", len(bad), "of", p.n_components)
for c in bad[:12]:
    nodes = p.comp_nodes[p.comp_ptr[c]:p.comp_ptr[c + 1]].astype(int)
    print(" slot", c, "nodes", sizes[c], "iters g/o", st_g["iterations"][c], st_o["iterations"][c], "term g/o", st_g["termination"][c], st_o["termination"][c],
          "cg_iters", int(cg[c]) if cta[c] else None, "cost g/o %.12g %.12g" % (st_g["final_cost"][c], st_o["final_cost"][c]), "maxerr %.2e" % np.abs(pos_g[nodes] - pos_o[nodes]).max())
ok = st_g["iterations"] == st_o["iterations"]
errs = []
for c in np.nonzero(ok & (sizes > 1))[0]:
    nodes = p.comp_nodes[p.comp_ptr[c]:p.comp_ptr[c + 1]].astype(int)
    errs.append(np.abs(pos_g[nodes] - pos_o[nodes]).max())
print("max err among matching-trajectory comps %.3e" % max(errs))
its = st_g["iterations"][cta]
print("CTA comps", cta.sum(), "cg iters per lm iteration: mean %.1f max %.1f" % ((cg[cta] / np.maximum(1, its)).mean(), (cg[cta] / np.maximum(1, its)).max()))
errs = np.zeros(p.n_components)
for c in range(p.n_components):
    nodes = p.comp_nodes[p.comp_ptr[c]:p.comp_ptr[c + 1]].astype(int)
    errs[c] = np.abs(pos_g[nodes] - pos_o[nodes]).max() if len(nodes) else 0
for c in np.argsort(-errs)[:6]:
    nodes = p.comp_nodes[p.comp_ptr[c]:p.comp_ptr[c + 1]].astype(int)
    nfree = int((~p.is_root[nodes].astype(bool)).sum())
    print(" worst-err slot", c, "nodes", sizes[c], "unknowns", 2 * nfree, "cta" if cta[c] else "warp", "iters g/o", st_g["iterations"][c], st_o["iterations"][c],
          "term", st_g["termination"][c], st_o["termination"][c], "ls", int(rec["ls_steps"][c]), "cost g/o %.14g %.14g" % (st_g["final_cost"][c], st_o["final_cost"][c]), "err %.2e" % errs[c])
