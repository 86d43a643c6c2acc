"""Worker of tests/test_gpu_step_exact.py for cases that need their own process (the fusion switches
CONVNET_B200_NO_FUSED_DROPOUT / _NO_DROPOUT_FOLD / _NO_PRESTAGE are read once per process):
    step_exact_worker.py MODEL BATCH MODE WARMUP
audits step number WARMUP and prints one ROW line per check, NAN lines for tensors the step left NaN in, then DONE."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import step_exact as se  # noqa: E402

model, batch, mode, warmup = sys.argv[1], int(sys.argv[2]), sys.argv[3], int(sys.argv[4])
rows, left, _ = se.audit_case(model, batch, mode, warmup)
for r in rows:
    print("ROW\t%s\t%s\t%d\t%.6e\t%s" % (r.layer, r.quantity, int(r.ok), r.worst, r.detail), flush=True)
for t in left:
    print("NAN\t%s" % t)
print("DONE")
