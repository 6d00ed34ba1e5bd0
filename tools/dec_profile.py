"""One hot-path-2 call at BASELINE configs[3] (64 x 469 tokens) between cudaProfilerStart/Stop, for

    ncu --profile-from-start off --metrics dram__bytes_read.sum,dram__bytes_write.sum,gpu__time_duration.sum \\
        --clock-control none --csv --log-file decoder_c4_dram.csv python tools/dec_profile.py

(the per-launch DRAM traffic of hot path 2).  With --summarise FILE it reads such a CSV and prints per-kernel totals
instead."""
import csv
import os
import sys
from collections import defaultdict

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def summarise(path):
    rows = [r for r in csv.reader(l for l in open(path) if l.startswith('"'))]
    hdr = rows[0]
    ik, im, iv, iid = hdr.index("Kernel Name"), hdr.index("Metric Name"), hdr.index("Metric Value"), hdr.index("ID")
    per = defaultdict(lambda: defaultdict(float))
    launches = defaultdict(set)
    for r in rows[1:]:
        name = r[ik].split("(")[0]
        per[name][r[im]] += float(r[iv].replace(",", ""))
        launches[name].add(r[iid])
    tot = defaultdict(float)
    print(f"{'kernel':60s} {'launches':>8s} {'ms':>9s} {'read MB':>10s} {'write MB':>10s}")
    for name, m in sorted(per.items(), key=lambda kv: -kv[1]["gpu__time_duration.sum"]):
        t, rd, wr = m["gpu__time_duration.sum"] / 1e6, m["dram__bytes_read.sum"] / 1e6, m["dram__bytes_write.sum"] / 1e6
        print(f"{name[:60]:60s} {len(launches[name]):8d} {t:9.3f} {rd:10.1f} {wr:10.1f}")
        tot["t"] += t; tot["rd"] += rd; tot["wr"] += wr
    print(f"{'TOTAL':60s} {sum(len(v) for v in launches.values()):8d} {tot['t']:9.3f} {tot['rd']:10.1f} {tot['wr']:10.1f}")
    print(f"dram bytes per call: {int((tot['rd'] + tot['wr']) * 1e6)}")


def main():
    if len(sys.argv) > 2 and sys.argv[1] == "--summarise":
        return summarise(sys.argv[2])
    import torch

    from chattts_b200.config import Config
    from chattts_b200.decoder import DVAE, Vocos
    from chattts_b200.synth import synth_dvae_state, synth_vocos_state

    B, T = 64, 469
    dev = torch.device("cuda", 0)
    cfg = Config()
    voc = Vocos(cfg.vocos, dev, max_batch=B, max_tokens=T)
    voc.state = synth_vocos_state(5)
    dec = DVAE(cfg.decoder, dim=cfg.decoder.idim, device=dev, vocos=voc, max_batch=B, max_tokens=T)
    dec.load_state_dict(synth_dvae_state(2, cfg.decoder, cfg.decoder.idim))
    x = torch.randn(B, T, 768, generator=torch.Generator().manual_seed(1)).to(dev)
    dec.engine.tokens_to_wav(x, 1)
    torch.cuda.synchronize()
    torch.cuda.cudart().cudaProfilerStart()
    w = dec.engine.tokens_to_wav(x, 1)
    torch.cuda.synchronize()
    torch.cuda.cudart().cudaProfilerStop()
    print("wav", tuple(w.shape), float(w.abs().mean()))


if __name__ == "__main__":
    main()
