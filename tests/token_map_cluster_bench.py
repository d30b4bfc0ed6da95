"""Time get_token_maps with the device spectral clustering against scikit-learn on the same affinity.

    python tests/token_map_cluster_bench.py [--reps 5] [--out DIR]

Affinities: the synthetic fixtures (tests/synth.synth_maps) and the capture of bench.py's config 2 shape (synthetic
SD1.5 UNet, plain CFG pass of 41 steps). For k = 4 and 9, spectral_clustering on the device affinity and
scikit-learn's SpectralClustering on its host copy (what get_token_maps ran before) are called alternately, followed by
the whole device get_token_maps; the device path is also split into Laplacian + eigh, host draws, the k-means kernel,
the copies back and the restart selection. Prints one JSON line per case and one with the card and host.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tests import synth  # noqa: E402


def sd15_capture():
    """[1024, 1024] device affinity of a plain 41-step CFG pass of the synthetic SD1.5 model (bench.py config 2), and
    the captured (self-attention, cross-attention) maps."""
    import bench
    from rtti_b200.attention_utils import self_affinity
    from rtti_b200.region_diffusion import RegionDiffusion
    cfg = bench.CONFIGS[2]
    model = RegionDiffusion.from_synthetic(seed=0, device=torch.device("cuda"), with_vae=False)
    wl = bench.synth_workload(cfg)
    ctx = wl["ctx"].cuda()
    model.register_tokenmap_hooks()
    with torch.no_grad():
        model.produce_attn_maps(None, None, num_inference_steps=cfg["schedule"], guidance_scale=bench.GUIDANCE,
                                latents=wl["latents"].cuda(), text_embeddings=torch.cat([ctx[:1], ctx[-1:]]), decode=False)
    maps = (dict(model.selfattn_maps), dict(model.crossattn_maps))
    model.remove_tokenmap_hooks()
    return self_affinity(maps[0]), maps


def _sync_t():
    torch.cuda.synchronize()
    return time.perf_counter()


def device_split(aff, k):
    """Seconds per stage of spectral_clustering's device path."""
    from rtti_b200 import attention_utils as au, ops
    t0 = _sync_t()
    emb, evals = au.spectral_embedding(aff, k)
    gap = float(evals[k] - evals[k - 1])
    t1 = _sync_t()
    rs = np.random.RandomState(0)
    rs.uniform(-1, 1, aff.shape[0])
    draws = au.kmeans_draws(rs, aff.shape[0], k, 100)
    draws_d = torch.from_numpy(draws).cuda()
    t2 = _sync_t()
    labels, inertia, n_iter, _ = ops.kmeans_fit(emb, draws_d)
    t3 = _sync_t()
    lab, ine = labels.cpu().numpy(), inertia.cpu().numpy()
    t4 = _sync_t()
    au.select_restart(lab, ine, k)
    t5 = time.perf_counter()
    return {"laplacian_eigh_s": t1 - t0, "host_draws_s": t2 - t1, "kernel_s": t3 - t2, "copies_s": t4 - t3,
            "select_s": t5 - t4, "eigengap": gap, "mean_lloyd_iters": float(n_iter.float().mean())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import subprocess
    from rtti_b200 import attention_utils as au
    name = torch.cuda.get_device_name()
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                                str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
    except OSError:
        power = "unknown"
    # warm-up: cuSOLVER handle / eigh workspace and the kernel module, each called directly
    from rtti_b200 import ops
    emb, _ = au.spectral_embedding(au.self_affinity({k: v.cuda() for k, v in synth.synth_maps(0)[0].items()}), 4)
    ops.kmeans_fit(emb, torch.from_numpy(au.kmeans_draws(np.random.RandomState(0), 1024, 4, 100)).cuda())
    torch.cuda.synchronize()

    obj = [torch.LongTensor([3]), torch.LongTensor([7, 8])]
    cases = []
    for s in range(2):
        selfm, crossm = synth.synth_maps(s)
        cases.append((f"synth{s}", {k: v.cuda() for k, v in selfm.items()}, {k: v.cuda() for k, v in crossm.items()}))
    _, (selfm, crossm) = sd15_capture()
    cases.append(("sd15_config2", selfm, crossm))
    results = []
    from sklearn.cluster import SpectralClustering
    for name_c, selfm, crossm in cases:
        aff = au.self_affinity(selfm)
        for k in (4, 9):
            dev_t, skl_t, gtm_t, same = [], [], [], True
            for _ in range(args.reps):
                t0 = _sync_t()
                np.random.seed(3)
                got = au.spectral_clustering(aff, k)
                t1 = _sync_t()
                np.random.seed(3)
                ref = SpectralClustering(k, affinity="precomputed", n_init=100, assign_labels="kmeans").fit_predict(
                    aff.cpu().numpy())
                t2 = _sync_t()
                au.get_token_maps(selfm, crossm, None, None, 64, 64, obj, seed=3, num_segments=k)
                t3 = _sync_t()
                dev_t.append(t1 - t0)
                skl_t.append(t2 - t1)
                gtm_t.append(t3 - t2)
                same &= bool(np.array_equal(got, ref))
            split = device_split(aff, k)
            results.append({"affinity": name_c, "k": k, "device_s_median": float(np.median(dev_t)),
                            "sklearn_s_median": float(np.median(skl_t)), "get_token_maps_s_median": float(np.median(gtm_t)),
                            "device_s": dev_t, "sklearn_s": skl_t, "labels_equal": same, "device_split": split,
                            "guard_fires": split["eigengap"] < au.EIGENGAP_MIN})
            print(json.dumps(results[-1]), flush=True)
    out = {"gpu": name, "power_limit": power, "host_threads": os.cpu_count(), "results": results}
    line = json.dumps({k: v for k, v in out.items() if k != "results"})
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "token_map_cluster_bench.json"), "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
