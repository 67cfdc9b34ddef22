"""Checks shared by the GPU tests of the float-distance, preemptive, Euclidean and LSC contexts: one class-API call
against the checker's outputs, and the kernel that call ran (Engine.dispatch())."""
import numpy as np

TMA, LDG, GENERIC, PREEMPT, LSC = 5, 4, 0, 13, 14  # Engine.DISPATCH_KERNELS
REAL_KERNELS = {"standard": 10, "l2": 11, "noq": 12}


def assert_kernel(name, d, kernel, max_iter):
    """Engine.dispatch() read-back `d` of one call shows that `kernel` ran: on every update pass (there are none at
    max_iter 0) and on the full pass -- except for the preemptive option, whose full pass is the ordinary one."""
    msg = "%s: the intended kernel %d did not run; read back %r" % (name, kernel, d)
    assert d["update"]["kernel"] == (kernel if max_iter > 0 else -1), msg
    assert d["full"]["kernel"] in ((TMA, LDG, GENERIC) if kernel == PREEMPT else (kernel,)), msg


def check_class_call(name, s, got, want, want_pre, cl, kernel, max_iter):
    """One iterate() of the class object `s` (labels `got`) against the checker: final labels, pre-CCA labels (read
    back from the cached context the call ran on), raw Cluster bytes and the kernel that ran."""
    from fast_slic_b200 import get_engine
    eng = get_engine(got.shape[0], got.shape[1], s.num_components, 1)
    pre = eng.debug_stages(1)[1][0].cpu().numpy().view(np.uint16)
    assert (pre == want_pre).all(), "%s: pre-CCA labels differ (%d px)" % (name, int((pre != want_pre).sum()))
    assert (got == want).all(), "%s: final labels differ (%d px)" % (name, int((got != want).sum()))
    assert s.slic_model.cluster_array.tobytes() == cl.tobytes(), "%s: Cluster bytes differ" % name
    assert_kernel(name, eng.dispatch(), kernel, max_iter)
