"""one-line digest of a bench.py JSON line: python tools/bench_brief.py TAG FILE"""
import json, sys
tag, path = sys.argv[1], sys.argv[2]
line = [l for l in open(path) if l.startswith("{")]
if not line:
    print(tag, "NO JSON LINE"); sys.exit(0)
d = json.loads(line[-1])
r = d.get("roofline") or {}
out = ["%-8s" % tag, "img/s %.0f" % d["value"], "ms %.4f" % d["ms_per_step"], "frac_burst %.3f" % r.get("frac_burst", 0)]
ek = r.get("edge_kernel_ms") or {}
out.append("conv1 %.4f dec_out %.4f" % (ek.get("enc_conv1", 0), ek.get("dec_out", 0)))
lm = r.get("layer_ms") or {}
out.append("gemm " + " ".join("%.3f" % lm[k] for k in lm))
if d.get("edit"):
    out.append("| edit %.0f (%.2f ms)" % (d["edit"]["value"], d["edit"]["ms_total"]))
f = d.get("full_ian")
if f and f.get("bf16"):
    out.append("| full bf16 %.0f (%.3f ms) fp32 %.0f" % (f["bf16"]["value"], f["bf16"]["ms_per_step"], (f.get("fp32_split") or {}).get("value", 0)))
    out.append("rgb_head %.3f conv4 %.3f" % (f["bf16"]["layer_ms"].get("rgb_head", 0), f["bf16"]["layer_ms"].get("full_dec_conv4", 0)))
if d.get("clocks"):
    out.append("| %s MHz %s W" % (d["clocks"].get("sm_mhz"), d["clocks"].get("power_w_max")))
print("  ".join(out))
