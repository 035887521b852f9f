"""Dev probe: mean device time of the attention kernel alone (not a bench line).  usage: attn_probe.py [B S W H mask iters]"""
import json
import sys

sys.path.insert(0, ".")
from marqo_b200.engine import debug_attention_time  # noqa: E402

cases = [(256, 257, 1024, 16, 0), (64, 512, 1024, 16, 2), (256, 128, 768, 12, 2), (256, 50, 768, 12, 0)]
if len(sys.argv) > 5:
    cases = [tuple(int(x) for x in sys.argv[1:6])]
iters = int(sys.argv[6]) if len(sys.argv) > 6 else 20
for B, S, W, H, mask in cases:
    ms = debug_attention_time(B, S, W, H, mask, iters=iters)
    flops = 4.0 * B * H * S * S * (W // H)
    print(json.dumps({"B": B, "S": S, "W": W, "H": H, "mask": mask, "us": ms * 1e3, "TFLOPs": flops / ms / 1e9}))
