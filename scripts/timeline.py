"""In-kernel timeline of one operator (CTA 0): python scripts/timeline.py qkv|attn|outproj_ln|ffn|tail|tail_fused [max_events]
Prints, per warp, the sequence of pipeline events with SM-clock deltas (cycles) from the kernel's first event."""
import ctypes as C, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from mld_b200 import synth, _lib
from mld_b200.engine import Engine, make_config

TAGS = {1: "prod:tile", 2: "mma:tile_begin", 3: "mma:tile_issued", 4: "epi:acc_ready", 5: "epi:drained", 6: "ln:res_issued", 7: "ln:stats_done", 17: "ln:merged", 18: "ln:stores_issued",
        10: "mma:F1_start", 11: "mma:F1_issued", 12: "mma:F2_start", 13: "e1:acc1_ready", 14: "e1:hs_written", 15: "ln:acc2_ready", 16: "ln:done",
        20: "prod:Q", 21: "prod:Vslot", 22: "mma:S_go", 23: "mma:K_landed", 24: "mma:S_issued", 25: "mma:P_written", 26: "mma:V_landed",
        40: "entry", 41: "pdl_waited", 42: "exit",
        50: "proj:item", 51: "proj:A_landed", 52: "proj:epi_begin", 53: "proj:epi_stored",
        60: "tail:outproj_kb", 61: "tail:ln1_done", 62: "tail:ln2_done", 63: "tail:y_store_read",
        30: "sm:wait_S", 31: "sm:S_ready", 32: "sm:pass1", 33: "sm:pass2", 34: "sm:O_ready", 35: "sm:epi_done"}
op = sys.argv[1] if len(sys.argv) > 1 else "attn"
maxe = int(sys.argv[2]) if len(sys.argv) > 2 else 400
eng = Engine(make_config(), 0)
eng.load_state_dict(synth.denoiser_state_dict(1234), "denoiser.")
eng.load_state_dict(synth.mld_vae_state_dict(4321), "vae.")
eng.finalize()
eng.set_timesteps(2)
eng.profile_op(op, 256, 77, 2)                       # warm
lib = _lib.lib()
_lib.check(lib.mldb_debug_timeline(1, None, 0, None))
eng.profile_op(op, 256, 77, 1)                       # 3 warm-up launches + 1 inside
cap = 16384
buf = (C.c_int64 * (2 * cap))()
n = C.c_int32()
_lib.check(lib.mldb_debug_timeline(0, buf, cap, C.byref(n)))
ev = [(buf[2 * i] & 0xffff, (buf[2 * i] >> 16) & 0xff, buf[2 * i] >> 24, buf[2 * i + 1]) for i in range(n.value)]
# every launch restarts the per-warp counters, so the slots hold the LAST launch (all launches log the same events)
ev.sort(key=lambda e: e[3])
t0 = ev[0][3]
print(f"op {op}: {len(ev)} events in the last launch, span {ev[-1][3] - t0} cycles")
by_warp = {}
for tag, warp, aux, t in ev:
    by_warp.setdefault(warp, []).append((t - t0, tag, aux))
for warp in sorted(by_warp):
    seq = by_warp[warp][:maxe]
    print(f"-- warp {warp} ({len(by_warp[warp])} events)")
    line, prev = [], 0
    for t, tag, aux in seq:
        line.append(f"{TAGS.get(tag, tag)}[{aux}]@{t}(+{t - prev})")
        prev = t
    for i in range(0, len(line), 6):
        print("   " + "  ".join(line[i:i + 6]))
