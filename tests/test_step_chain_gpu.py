"""A tracking step's kernels run as one dependent-launch chain (DESIGN §3.4): the next frames' cache store may start under the last
tails of the k_solve that read the same slots, and k_prep_frames / k_solve under their predecessors.  These tests run bench.py's step
pattern - the same cache slots rewritten every step right behind the solve that read them - and require the poses to be byte-identical
to the same sequence with the device synchronised after every library call, where no two kernels can overlap."""
import numpy as np
import pytest

from bundletrack_b200 import synth

pytestmark = pytest.mark.gpu
N_WIN, N_FR = 8, 10


@pytest.fixture(scope="module")
def scenes(cuda_device):
    import torch
    out = []
    for s in range(4):
        w = synth.make_window(900 + s, n_frames=N_FR, n_corr=800)
        d = [torch.from_numpy(np.ascontiguousarray(w.depth[f])).to(cuda_device) for f in range(N_FR)]
        n = [torch.from_numpy(np.ascontiguousarray(w.normal[f])).to(cuda_device) for f in range(N_FR)]
        out.append((w, d, n))
    return out


def _sequence(scenes, cuda_device, timing, all_frames, sync):
    """Poses the solves of a fixed call sequence produced.  `all_frames`: every step stores all 80 frames of the batch (the store
    with uploaded tables) instead of one new frame per window (the tables in the kernel parameters)."""
    import torch
    from bundletrack_b200.optimizer import OptimizerGpu, SolveWindow
    stream = torch.cuda.current_stream().cuda_stream
    opt = OptimizerGpu(None, device=0, max_windows=N_WIN, max_frames=N_FR, max_corr=800, stream=stream)
    opt.enable_timing(timing)
    wins = [scenes[k % len(scenes)] for k in range(N_WIN)]
    w0 = wins[0][0]
    opt.reserve_frame_cache(N_WIN * N_FR, w0.H, w0.W)
    slots = list(range(N_WIN * N_FR))
    # two versions of the rewritten frames: a window's own maps, and the maps of the next scene's frames (other poses come out)
    if all_frames:
        st_slots = slots
        maps = [([d for w, ds, _ in wins for d in ds], [n for w, _, ns in wins for n in ns]),
                ([d for k in range(N_WIN) for d in wins[(k + 1) % N_WIN][1]], [n for k in range(N_WIN) for n in wins[(k + 1) % N_WIN][2]])]
    else:
        st_slots = [k * N_FR + N_FR - 1 for k in range(N_WIN)]
        maps = [([ds[N_FR - 1] for _, ds, _ in wins], [ns[N_FR - 1] for _, _, ns in wins]),
                ([ds[N_FR - 2] for _, ds, _ in wins], [ns[N_FR - 2] for _, _, ns in wins])]
    stores = [opt.prepare_store(st_slots, d, n, w0.H, w0.W, w0.K) for d, n in maps]
    opt.store_frames(slots, [d for _, ds, _ in wins for d in ds], [n for _, _, ns in wins for n in ns], w0.H, w0.W, w0.K)
    cw = [SolveWindow(w.corr, w.H, w.W, None, None, w.poses_init, w.K, cache_slots=slots[k * N_FR:(k + 1) * N_FR]) for k, (w, _, _) in enumerate(wins)]

    def call(f, *a):
        r = f(*a)
        if sync:
            torch.cuda.synchronize()
        return r

    out = []
    opt.stage(cw)
    for k in range(6):      # bench's value loop; every other step the solve's poses are read after the next store rewrote its slots
        call(opt.store_prepared, stores[k % 2])
        call(opt.run)
        if k % 2:
            call(opt.store_prepared, stores[(k + 1) % 2])
            out.append(np.concatenate(opt.fetch(), 0))
    for k in range(3):      # store + run back to back, then the last solve's poses
        call(opt.store_prepared, stores[k % 2])
        call(opt.run)
    out.append(np.concatenate(opt.fetch(), 0))
    # bench's e2e loop: the streaming calls, two batches in flight, the slots rewritten between them
    batch = opt.prepare_batch(cw)
    buf = np.empty((batch.poses.shape[0], 4, 4), np.float32)
    for k in range(5):
        call(opt.store_prepared, stores[k % 2])
        call(opt.begin_prepared, batch)
        if k:
            opt.end_prepared(batch, buf)
            out.append(buf.copy())
    opt.end_prepared(batch, buf)
    out.append(buf.copy())
    # the resident-input loop once more after the streaming calls (the staging blocks have turned over)
    opt.stage(cw)
    for k in range(2):
        call(opt.store_prepared, stores[k % 2])
        call(opt.run)
    out.append(np.concatenate(opt.fetch(), 0))
    if timing:
        tm = opt.timing_ms()
        assert tm["prep"] > 0 and tm["plan"] >= 0 and tm["solve"] > 0, tm
    opt.close()
    return out


@pytest.mark.parametrize("all_frames", [False, True], ids=["inline_tables", "uploaded_tables"])
@pytest.mark.parametrize("timing", [False, True], ids=["timing_off", "timing_on"])
def test_chained_steps_equal_synchronised_steps(scenes, cuda_device, timing, all_frames):
    chained = _sequence(scenes, cuda_device, timing, all_frames, sync=False)
    ref = _sequence(scenes, cuda_device, timing, all_frames, sync=True)
    assert len(chained) == len(ref)
    for k, (a, b) in enumerate(zip(chained, ref)):
        assert np.isfinite(b).all()
        assert a.tobytes() == b.tobytes(), f"result {k} differs from the synchronised sequence"
    # the two versions of the rewritten frames give different poses (results 0 and 3), so a solve that read the wrong version would show
    assert ref[0].tobytes() != ref[3].tobytes()
