"""The library's run-time knobs (tb_kernels.cuh: Knobs), the environment variables a renderer reads when it is created.
Every variant they select gives the same bits, so a test that means to check one route must set exactly the knobs
that name it and clear the rest: `knobs` does that, and the GPU tests set these variables through it alone."""
import contextlib
import os

PREFIX = "TINSEL_B200_"
KEYS = ("TINSEL_B200_PIPELINE", "TINSEL_B200_READBACK", "TINSEL_B200_TEST_LAUNCH_SAMPLES", "TINSEL_B200_TEST_DUP_DEVICES",
        "TINSEL_B200_SCHED", "TINSEL_B200_SPLIT", "TINSEL_B200_CTA", "TINSEL_B200_QUEUES", "TINSEL_B200_SPECIALIZE",
        "TINSEL_B200_NO_FLAT", "TINSEL_B200_TREELET")

# Route settings, by the names the tests give them.  "lanes" is the lane-owned layout whatever the launch and mesh
# size: free-running scheduler, 512-thread CTAs, no split trace queue.
LANES = dict(QUEUES="lanes", SCHED="free", CTA="512", SPLIT="0")
ROUTES = {
    "mega": dict(PIPELINE="mega"),
    "wavefront": {},
    "lanes": LANES,
    "rings": dict(QUEUES="ring"),
    "lanes-generic": dict(LANES, SPECIALIZE="0"),
    "no-flat": dict(NO_FLAT="1"),
}

CTAS = ["512", "768"]
SCHEDS = ["hard", "free", "ring", "split", "treelet"]


@contextlib.contextmanager
def knobs(**settings):
    """Runs the body with the knobs named here (without the prefix: knobs(QUEUES="lanes")) set and every other one
    unset; None also means unset.  Yields the settings in force, as strings.  Restores the environment on exit."""
    unknown = [k for k in settings if PREFIX + k not in KEYS]
    assert not unknown, "not a library knob: %s" % unknown
    applied = {k: str(v) for k, v in settings.items() if v is not None}
    saved = {k: os.environ.pop(k, None) for k in KEYS}
    os.environ.update({PREFIX + k: v for k, v in applied.items()})
    try:
        yield applied
    finally:
        for k, v in saved.items():
            os.environ.pop(k, None)
            if v is not None:
                os.environ[k] = v


def sched_knobs(sched, cta, no_flat=False):
    """The settings of one scheduler variant: hard phases; free running; free running with the ring queues, the split
    trace queue forced on for every scene that has a mesh, or the top of the biggest mesh's BVH staged in shared memory
    for the inline walk ("treelet").  no_flat: the scene level always runs the reference-order walk."""
    return dict(SCHED="free" if sched in ("split", "treelet", "ring") else sched,
                QUEUES="ring" if sched == "ring" else "lanes",
                TREELET="1" if sched == "treelet" else "0",
                SPLIT="1" if sched == "split" else "0",
                CTA=cta,
                NO_FLAT="1" if no_flat else None)


def sched_env(sched, cta, no_flat=False):
    return knobs(**sched_knobs(sched, cta, no_flat))
