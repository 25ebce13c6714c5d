"""Plain-Python restatement of the launch plan and the in-kernel branches of the fused integer-grid attention
(csrc/int8_attention.cu), in the manner of tests/int8_geometry.py: given a call's shapes and options, ``branches``
names the kernel paths the call reaches, so that the cases of tests/test_gpu_int8_attention_branches.py can be tied
to the branch each exists for and a CPU test can check that together they reach every branch.  When the .cu file
changes, this file has to follow.  Line numbers are of csrc/int8_attention.cu.

There is one kernel and one way through it: K and v^T are streamed through the ring in both passes (no resident
variant was built), so the branches are the tails, the block counts and the options."""
from int8_geometry import cdiv

ROWS = 128          # :33 kAtRows, query rows per CTA
KEYS = 128          # :34 kAtKeys, keys per block
STAGES = 4          # :35 kAtStages
MAX_DIM = 128       # :40 kAtMaxDim
MAX_TK = 1 << 17    # :41 kAtMaxTk

ALL = ("q_tail", "q_full_tile", "q_many_tiles", "key_tail", "key_full_block", "one_key_block", "many_key_blocks",
       "ring_wraps", "k16_pad", "d_steps_lt4", "d_steps_4", "dv_tail", "dv_full", "dv_odd_scalar", "dv_even_vec2",
       "p_q_on", "p_q_off", "scale_on", "scale_off", "max_rescaled", "exp_underflow",
       "nan_q", "nan_k", "nan_v")


def plan(batch, tq, tk, d, dv):
    """The host side, :323-335 and :373-417: None when the call is rejected, else the launch values."""
    if min(batch, tq, tk, d, dv) <= 0 or d > MAX_DIM or dv > MAX_DIM or tk >= MAX_TK:
        return None
    dp, tkp = cdiv(d, 16) * 16, cdiv(tk, 16) * 16
    return dict(ctas=batch * cdiv(tq, ROWS), nkb=cdiv(tk, KEYS), nk32=cdiv(dp, 32), dp=dp, tkp=tkp)


def branches(batch, tq, tk, d, dv, p_q=True, scale=None, p_signed=False, ramp=False, spread=False, nan=()):
    """The branch names a call reaches.  ``p_signed`` is not a branch: it only sets p's stored offset and clamp
    bounds on the host (:408-409); the cases still run both.  ``ramp``: the scores of a later key block exceed every earlier one (the
    running max is rescaled, :183-186); ``spread``: some exp(s - m) underflows (:65); ``nan``: which operands hold a
    NaN."""
    p = plan(batch, tq, tk, d, dv)
    out = set()
    out.add("q_tail" if tq % ROWS else "q_full_tile")            # :240, :282 rows past Tq are not stored
    if tq > ROWS:
        out.add("q_many_tiles")                                   # :96-97 m0 = (blockIdx % tiles_q) 128
    out.add("key_tail" if tk % KEYS else "key_full_block")        # :171, :229 keys past Tk are masked
    out.add("one_key_block" if p["nkb"] == 1 else "many_key_blocks")  # :157, :213
    if 2 * p["nkb"] > STAGES:
        out.add("ring_wraps")                                     # :154, :205, :275 stage reuse with alternating parity
    if tk % 16:
        out.add("k16_pad")                                        # :240 p_q padding, v^T padding in [Tk, Tkp)
    out.add("d_steps_lt4" if p["nk32"] < 4 else "d_steps_4")      # :77 k32 steps past dp are skipped
    out.add("dv_tail" if dv < MAX_DIM else "dv_full")             # :272 columns past dv
    out.add("dv_even_vec2" if dv % 2 == 0 else "dv_odd_scalar")   # :290-295
    out.add("p_q_on" if p_q else "p_q_off")                       # :240
    out.add("scale_on" if scale is not None else "scale_off")     # :174, :232
    if ramp and p["nkb"] > 1:
        out.add("max_rescaled")                                   # :183-186
    if spread:
        out.add("exp_underflow")                                  # :65
    out.update(f"nan_{o}" for o in nan)                           # :148, :205, :278
    return out
