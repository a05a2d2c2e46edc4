"""Constants shared by the tests of ggufb200_linear_fallback (the Linear of the numpy-fallback types) on the CPU and the GPU."""
from fallback_cases import FALLBACK

Q = FALLBACK[0].__class__
# AUTO's crossover M (csrc/api.cu, fallback_crossover): FUSED_SYNC up to it where the kernel splits K (`auto_fused`),
# DEQUANT_MMA above it; TQ1_0 never takes FUSED_SYNC
CROSSOVER = {q: {Q.TQ1_0: 0, Q.TQ2_0: 32, Q.MXFP4: 32, Q.NVFP4: 32}.get(q, 64) for q in FALLBACK}
# the H100's SM count, which the split-K plan assumes when no device is visible (common.cuh sm_count)
SMS_NO_DEVICE = 132
# the kernel's tile (csrc/linear_fallback.cu): features and tokens per CTA, k per K step; the plan's limits on K ranges
FEATURES_PER_CTA, TOKENS_PER_CTA, K_STEP, MIN_STEPS, MAX_SPLITS = 128, 64, 128, 4, 16


def tiles(M, N):
    return -(-N // FEATURES_PER_CTA) * -(-M // TOKENS_PER_CTA)


def splits_of(ws, M, N):
    """K ranges of a FUSED_SYNC plan from its workspace (ggufb200_linear_fallback_workspace): fp32 [splits, M, N], 0 unsplit."""
    assert ws % (M * N * 4) == 0, (ws, M, N)
    return max(1, ws // (M * N * 4))


def plan_problems(M, N, K, ws, sms=SMS_NO_DEVICE):
    """What is wrong with a FUSED_SYNC plan, as properties rather than a restatement of the planner: a grid that fills the SMs
    runs unsplit; a split never launches more CTAs than SMs, never gives a range fewer than MIN_STEPS steps on average, and
    stays within MAX_SPLITS; a grid that fills at most half the SMs, with K long enough for two ranges, is split."""
    if ws % (M * N * 4):
        return [f"workspace {ws} is not whole [M, N] fp32 slices"]
    s, t, steps = splits_of(ws, M, N), tiles(M, N), -(-K // K_STEP)
    bad = []
    if s == 1 and ws != 0:
        bad.append("one K range but a workspace")
    if t >= sms and s > 1:
        bad.append(f"{t} tiles fill the SMs, yet {s} ranges")
    if s > 1 and (t * s > sms or s > MAX_SPLITS or s * MIN_STEPS > steps):
        bad.append(f"{s} ranges for {t} tiles, {steps} steps")
    if 2 * t <= sms and steps >= 2 * MIN_STEPS and s < 2:
        bad.append(f"{t} tiles fill at most half the SMs and K has {steps} steps, yet unsplit")
    return bad


def auto_fused(qt, M, fused_ws):
    """AUTO takes FUSED_SYNC: M up to the type's crossover, and the kernel's plan (its workspace) cuts K into ranges."""
    return M <= CROSSOVER[qt] and fused_ws > 0
