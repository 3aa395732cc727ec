"""The wavefront kernel's scheduler variants, selected through environment variables: every variant must give
the same bits.  Shared by the parity tests over fixed scenes and the mesh fuzz."""
import contextlib
import os

CTAS = ["512", "768"]
SCHEDS = ["hard", "free", "ring", "split", "treelet", "offload", "offload1", "offload100"]
KEYS = ("TINSEL_B200_SCHED", "TINSEL_B200_SPLIT", "TINSEL_B200_CTA", "TINSEL_B200_OFFLOAD", "TINSEL_B200_WALKERS", "TINSEL_B200_TREELET",
        "TINSEL_B200_QUEUES", "TINSEL_B200_NO_FLAT")


@contextlib.contextmanager
def sched_env(sched, cta, no_flat=False):
    """hard phases; free running; free running with the ring queues, the split trace queue forced on for every
    scene that has a mesh, or the top of the biggest mesh's BVH staged in shared memory for the inline walk
    ("treelet"); the mesh-walk offload forced on for every mesh with the default number of walker CTAs, a
    single one, and as many as fit.  no_flat: the scene level always runs the reference-order walk."""
    offload = sched.startswith("offload")
    os.environ["TINSEL_B200_SCHED"] = "free" if sched in ("split", "treelet", "ring") or offload else sched
    os.environ["TINSEL_B200_QUEUES"] = "ring" if sched == "ring" else "lanes"
    os.environ["TINSEL_B200_TREELET"] = "1" if sched == "treelet" else "0"
    os.environ["TINSEL_B200_SPLIT"] = "1" if sched == "split" else "0"
    os.environ["TINSEL_B200_OFFLOAD"] = "2" if offload else "0"
    if sched in ("offload1", "offload100"):
        os.environ["TINSEL_B200_WALKERS"] = sched[len("offload"):]
    os.environ["TINSEL_B200_CTA"] = cta
    if no_flat:
        os.environ["TINSEL_B200_NO_FLAT"] = "1"
    try:
        yield
    finally:
        for k in KEYS:
            os.environ.pop(k, None)
