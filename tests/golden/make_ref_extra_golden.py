"""Generates the fixtures that let the remaining comparisons with the reference's own code run without it:

  ref_extra_golden.json   digests of the reference's maps on the fuzz cases (tests/fuzz_cases.py) and after the 10 012-frame
                          full-reset sequence, its ros_params.cpp output on the parameter cases of tests/test_shim_cpu.py, and the
                          label tables its CSV reader builds from the label files it ships (copied to label_csv/)
  ref_base_helpers.npz    its SemanticIntegratorBase helpers on the seeded vectors of test_host_helpers_of_the_shim_...

Everything comes from oracle/_ref (the reference's sources compiled against the stand-in headers, `make -C oracle ref`).
Regenerate where the reference sources are present:   make -C oracle ref && python tests/golden/make_ref_extra_golden.py
"""
import json
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, HERE)
import numpy as np  # noqa: E402

import fuzz_cases  # noqa: E402
import make_ref_golden as mrg  # noqa: E402
from oracle import ref_py  # noqa: E402

CSV_DIR = os.path.join(HERE, "label_csv")
PARAM_CASES = [   # (parameter lines without the CSV path; the cases of test_params_reader_equals_the_reference_ros_params)
    "method: merged\nsemantic_color_mode: semantic_probability\nsemantic_measurement_probability: 0.75\ndynamic_semantic_labels: [20, 3, 7]\n",
    "dynamic_semantic_labels: []\n",
    "semantic_color_mode: rainbow\ndynamic_semantic_labels: [1]\n",
    "method: fast\n",
]
SMALL_CSV = "name,red,green,blue,alpha,id\nfloor,10,20,30,255,1\nwall,40,50,60,255,2\n"


def helper_inputs():
    """The seeded vectors of the base-helper comparison: (config, priors [n, C], one-hot / count frequencies [n, C])."""
    cfg = mrg.case_config("fast_p08")
    C, n = 21, 200
    rng = np.random.default_rng(7)
    priors = (-rng.uniform(0.1, 40.0, (n, C))).astype(np.float32)
    freqs = rng.integers(0, 6, (n, C)).astype(np.float32)
    freqs[::5] = np.eye(C, dtype=np.float32)[rng.integers(0, C, len(freqs[::5]))]      # one-hot rows, as `fast` produces them
    return cfg, priors, freqs


def tiny_frames(n_frames, points_per_frame=24, seed=5):
    """Many tiny clouds: drives the ApproxHashSet offset through its full-reset threshold (A.4: 10 000 resets)."""
    from kimera_semantics_b200 import synth
    rng = np.random.default_rng(seed)
    for f in range(n_frames):
        T = synth.pose(f % 300)
        xyz = np.stack([rng.uniform(-0.4, 0.4, points_per_frame), rng.uniform(-0.3, 0.3, points_per_frame),
                        rng.uniform(0.8, 1.6, points_per_frame)], axis=1).astype(np.float32)
        lab = rng.integers(0, 20, points_per_frame).astype(np.uint8)
        yield T, xyz, lab


def full_reset_config():
    from kimera_semantics_b200.capi import KSG_INTEGRATOR_FAST
    from parity_utils import make_config
    return make_config(KSG_INTEGRATOR_FAST, 0.10, 21, max_points=64)


def run_params(text):
    """ros_params.cpp in its own process (it aborts on a fatal error) -> {"ok", "out" (CSV path as {csv}) | "fatal" (message)}."""
    with tempfile.TemporaryDirectory() as td:
        csv = os.path.join(td, "labels.csv")
        open(csv, "w").write(SMALL_CSV)
        r = subprocess.run([sys.executable, "-c", "import sys; from oracle import ref_py; sys.stdout.write(ref_py.ros_params(sys.stdin.read()))"],
                           input=text + f"semantic_label_2_color_csv_filepath: {csv}\n", capture_output=True, text=True, cwd=ROOT)
        if r.returncode == 0:
            return {"ok": True, "out": r.stdout.replace(csv, "{csv}")}
        last = [l for l in r.stderr.splitlines() if l.strip()][-1]
        return {"ok": False, "fatal": last.split("] ", 1)[-1]}


def run_csv(path):
    """The reference's CSV reader in its own process (it aborts on a malformed file) -> {"ok", "dump" | "fatal"}."""
    r = subprocess.run([sys.executable, "-c", "import sys; from oracle import ref_py; sys.stdout.write(ref_py.csv_dump(sys.argv[1]))", path],
                       capture_output=True, text=True, cwd=ROOT)
    if r.returncode == 0:
        return {"ok": True, "dump": r.stdout}
    last = [l for l in r.stderr.splitlines() if l.strip()][-1]
    return {"ok": False, "fatal": last.split("] ", 1)[-1]}


def main():
    assert ref_py.available(), "build oracle/_ref first: make -C oracle ref"
    out = {"fuzz": {}, "params": [run_params(t) for t in PARAM_CASES], "label_csv": {}}
    with fuzz_cases.quiet_stderr():
        for seed in range(24):
            cfg, frames = fuzz_cases.make_case(seed)
            ref = ref_py.RefHybridIntegrator(cfg)
            for T, pts, rgba, freespace in frames:
                ref.integrate_points(T, pts, rgba=rgba, freespace=freespace)
            out["fuzz"][str(seed)] = mrg.digest(ref.export())
        cfg = full_reset_config()
        pal = np.array([[cfg.label_color[l][k] for k in range(4)] for l in range(256)], np.uint8)
        ref = ref_py.RefHybridIntegrator(cfg)
        for T, xyz, lab in tiny_frames(10012):
            ref.integrate_points(T, xyz, rgba=np.ascontiguousarray(pal[lab]))
        out["full_reset_10012"] = mrg.digest(ref.export())
    for name in sorted(os.listdir(CSV_DIR)):
        out["label_csv"][name] = run_csv(os.path.join(CSV_DIR, name))
    json.dump(out, open(os.path.join(HERE, "ref_extra_golden.json"), "w"), indent=1, sort_keys=True)

    cfg, priors, freqs = helper_inputs()
    ref = ref_py.RefHybridIntegrator(cfg)
    L, lm, ln = ref.log_likelihood()
    upd = np.stack([ref.update_probabilities(freqs[k], priors[k]) for k in range(len(priors))])
    np.savez_compressed(os.path.join(HERE, "ref_base_helpers.npz"), log_likelihood=L, lm=np.float32(lm), ln=np.float32(ln), updated=upd,
                        label_rgba=np.stack([ref.label_color(l) for l in range(21)]),
                        normalized=np.stack([ref.normalize_probabilities(u) for u in upd]))
    print("wrote", os.path.join(HERE, "ref_extra_golden.json"), "and ref_base_helpers.npz")


if __name__ == "__main__":
    main()
