"""Peak device memory of one RAFT call per correlation plan: the measurement behind RAFT_WS_BYTES_PER_PX and
OTF_BYTES_PER_PAIR_PX in propainter_b200/RAFT/raft.py.

  python profiles/raft_mem.py [OUT.json]

All-pairs: peak above the inputs of a 2-frame call (one pair per direction) minus its two pyramids, per input pixel of
the two frames.  On-the-fly: slope of the peak between 2- and 4-frame calls (4 more pairs, 2 more frames encoded), per
added pair and input pixel.  Eager calls (no graph), 20 iterations, random-init weights; card name and power limit are
read in the same run."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import torch
    import __graft_entry__ as g
    g.build()
    from propainter_b200 import synth
    from propainter_b200.model.modules.flow_comp_raft import RAFT_bi
    from propainter_b200.RAFT.raft import ALL_PAIRS, ON_THE_FLY, pyramid_bytes
    dev = torch.device("cuda:0")
    raft = RAFT_bi(None, dev, seed=1).fix_raft

    def peak(T, H, W, plan):
        u8, _, _ = synth.make_clip(T, H, W, seed=3)
        fr = (torch.from_numpy(u8).to(dev).permute(0, 3, 1, 2).float() / 127.5 - 1).contiguous()
        raft._flows_bidirectional(fr, 20, plan)                 # weights packed, cuDNN plans chosen
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats(dev)
        base = torch.cuda.memory_allocated(dev)
        raft._flows_bidirectional(fr, 20, plan)
        torch.cuda.synchronize()
        return torch.cuda.max_memory_allocated(dev) - base

    out = {"card": torch.cuda.get_device_name(dev),
           "power_limit_w": subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                                           capture_output=True, text=True).stdout.strip()}
    for H, W in ((720, 1280), (1080, 1920)):
        p = peak(2, H, W, ALL_PAIRS)
        pyr = 2 * pyramid_bytes(H // 8, W // 8)
        p2, p4 = peak(2, H, W, ON_THE_FLY), peak(4, H, W, ON_THE_FLY)
        out[f"{W}x{H}"] = {"all_pairs_peak": p, "pyramids": pyr, "all_pairs_ws_bytes_per_px": (p - pyr) / (2 * H * W),
                           "otf_peak_2f": p2, "otf_peak_4f": p4, "otf_bytes_per_pair_px": (p4 - p2) / (4 * H * W),
                           "otf_peak_2f_per_pair_px": p2 / (2 * H * W)}
    print(json.dumps(out, indent=1))
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
