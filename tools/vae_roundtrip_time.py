"""Round-trip time of the full auto-encoders with a sampled posterior (the VAE trainers' forward shape): AutoencoderKL at
4096 faces of 32 x 32 and AutoencoderKL1D at 65 536 edges of 32 points, random-init weights, one GPU.

    python tools/vae_roundtrip_time.py            # env: FACES, EDGES, ROUNDS, ITERS

Two arms per network, alternated in one process (ROUNDS rounds of ITERS calls each, CUDA events, median per arm):
  fused    forward(x, sample_posterior=True): one bg_vae_reconstruct per chunk (encoder, posterior, decoder on the device)
  unfused  encode(x).latent_dist (bg_vae_encode_moments) -> the posterior as torch ops (mean + exp(0.5 logvar) * noise)
           -> decode(z)
Both arms draw their noise from the same seeded CUDA generator, and the script prints the relative L2 difference of the
two reconstructions next to the times (the torch posterior rounds mean + std * noise separately, the kernel with one FMA)."""
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from brepgen_b200.spec import edge_decoder_spec, edge_encoder_spec, surf_decoder_spec, surf_encoder_spec  # noqa: E402
from brepgen_b200.synth import synth_state_dict  # noqa: E402
from brepgen_b200.vae import AutoencoderKL, AutoencoderKL1D, randn_tensor  # noqa: E402

FACES = int(os.environ.get("FACES", 4096))
EDGES = int(os.environ.get("EDGES", 65536))
ROUNDS = int(os.environ.get("ROUNDS", 5))
ITERS = int(os.environ.get("ITERS", 3))


def gpu_info() -> str:
    try:
        q = "name,power.limit,clocks.sm,clocks.max.sm"
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except Exception as e:   # the numbers are still printed, without the clock reading
        return f"{torch.cuda.get_device_name(0)} (nvidia-smi unavailable: {e})"


def fused(m, x, seed):
    return m(x, sample_posterior=True, generator=torch.Generator(device="cuda").manual_seed(seed)).sample


def unfused(m, x, seed):
    post = m.encode(x).latent_dist
    noise = randn_tensor(post.mean.shape, generator=torch.Generator(device="cuda").manual_seed(seed), device=x.device,
                         dtype=torch.float32)
    z = post.mean + torch.exp(0.5 * torch.clamp(post.parameters[:, 3:], -30.0, 20.0)) * noise
    return m.decode(z).sample


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(ITERS):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / ITERS


def main():
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(0)
    cases = []
    for name, cls, specs, x in (
            ("AutoencoderKL", AutoencoderKL, (surf_encoder_spec(), surf_decoder_spec()),
             torch.rand(FACES, 3, 32, 32, generator=g) * 2 - 1),
            ("AutoencoderKL1D", AutoencoderKL1D, (edge_encoder_spec(), edge_decoder_spec()),
             torch.rand(EDGES, 3, 32, generator=g) * 2 - 1)):
        m = cls()
        m.load_state_dict({**synth_state_dict(specs[0], 3), **synth_state_dict(specs[1], 3)}, strict=True)
        cases.append((name, m.to(dev).eval(), x.to(dev)))
    print(f"GPU: {gpu_info()}", flush=True)
    with torch.no_grad():
        for name, m, x in cases:
            a, b = fused(m, x, 1), unfused(m, x, 1)            # warm-up: handles, workspaces, captured chunk graphs
            torch.cuda.synchronize()
            diff = float((a.double() - b.double()).norm() / b.double().norm())
            t = {"fused": [], "unfused": []}
            for _ in range(ROUNDS):
                t["fused"].append(timed(lambda: fused(m, x, 1)))
                t["unfused"].append(timed(lambda: unfused(m, x, 1)))
            mf, mu = statistics.median(t["fused"]), statistics.median(t["unfused"])
            print(f"{name} N={x.shape[0]}: fused {mf:.1f} ms (min {min(t['fused']):.1f}, max {max(t['fused']):.1f})  "
                  f"unfused {mu:.1f} ms (min {min(t['unfused']):.1f}, max {max(t['unfused']):.1f})  "
                  f"unfused/fused {mu / mf:.3f}  rel_l2(fused, unfused) {diff:.2e}", flush=True)
    print(f"GPU after: {gpu_info()}", flush=True)


if __name__ == "__main__":
    main()
