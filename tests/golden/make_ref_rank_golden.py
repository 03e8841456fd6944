"""Generate tests/golden/ref_rank_golden_*.pt (the cases of rank_cases.py, LoRA ranks 24, 96 and 128) by running the REFERENCE's OWN
code, exactly as make_ref_model_golden.py does for the rank-4 cases (build container only; needs /root/reference):

    python tests/golden/make_ref_rank_golden.py

Each case goes through make_ref_model_golden.run_case: the reference's model classes, `BaseTrainer.add_lora_adapter` with the case's
`r` / `lora_alpha`, its trainers' `_compute_loss` and losses, with `diffusers` / `peft` / `accelerate` replaced by tests/shims.  The
GPU machine never runs this; it reads the committed .pt files.
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_ref_model_golden as gen  # noqa: E402  (installs the shims and imports the reference)
import rank_cases  # noqa: E402


def main():
    out = {}
    for name, spec in rank_cases.RANK_CASES.items():
        out[name] = gen.run_case(name, spec)
        c = out[name]
        print(f"{name:28s} r={spec['r']} loss={float(c['loss']):.6f} pred={tuple(c['pred'].shape)} n_lora={len(c['grads'])} "
              f"|g|={float(sum(g.norm() ** 2 for g in c['grads'].values()) ** 0.5):.4e}")
    for path in rank_cases.save(out, HERE, "ref_rank_golden"):
        print("wrote", path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()
