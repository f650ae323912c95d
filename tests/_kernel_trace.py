"""The CUDA kernels a piece of work launches, by ``torch.profiler``, for the tests that pin an agent step's launch list."""
import torch


def profiled_kernels(window, required, warmup=True, attempts=5):
    """Names of the CUDA kernels (Memcpy / Memset left out) that one call of ``window()`` launches.  ``warmup``: one call is
    a profiler warm-up cycle and the next one is recorded (events launched as the tracer starts can be missed).

    The profiler at times loses kernel records of a session -- some of them or all of them -- in a process that has
    profiled before.  A lost record can only lower a count, never raise one.  So when a kernel of ``required`` (name
    substring -> how many the caller asserts) shows up fewer times than that, the window is profiled again, at most
    ``attempts`` times in all.  A kernel the work really fails to launch is missing from every session.  An extra or
    foreign kernel is never profiled again.  The caller checks whatever list is returned, exactly as before."""
    cuda = [torch.profiler.ProfilerActivity.CUDA]
    kernels = []
    for _ in range(attempts):
        if warmup:
            sched = torch.profiler.schedule(wait=0, warmup=1, active=1, repeat=1)
            with torch.profiler.profile(activities=cuda, schedule=sched) as prof:
                for _ in range(2):
                    window()
                    prof.step()
        else:
            with torch.profiler.profile(activities=cuda) as prof:
                window()
        kernels = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
                   and not e.name.startswith(("Memcpy", "Memset"))]
        if all(sum(name in k for k in kernels) >= n for name, n in required.items()):
            break
    return kernels
