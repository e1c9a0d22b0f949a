"""Big-int model of b2g_verify_batch_keys (csrc/verify.cu), shared by tests/test_batch_keys_model.py (CPU) and
tests/test_verify_batch_keys.py (GPU).  TEST INFRASTRUCTURE ONLY.  The keyed call checks b2g_verify_batch's equation once per
key over that key's proofs, so its model is tests/batch_model.py's verify_batch_rlc taken per key."""
from batch_model import verify_batch_rlc


def verify_batch_keys_rlc(batches, weights) -> list:
    """one verdict per (pvk, public_inputs, proofs) batch with its weights: verify_batch_rlc of the batch, True when it is
    empty"""
    return [verify_batch_rlc(pvk, ins, prs, w) if prs else True for (pvk, ins, prs), w in zip(batches, weights)]
