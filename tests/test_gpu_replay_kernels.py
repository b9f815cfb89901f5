"""The replay-memory kernels of csrc/b2q_rpm.cu against exact references: both samplers gather exactly ring[slot] for the slot formula of
tests/es_ref.py (bit for bit, all five arrays), with both seed conventions pinned; the plain, cursor and masked appends equal a torch ring
model at row widths on both sides of the CTAs' 64- and 32-wide strides; and the masked append is exercised at sizes where one CTA
copies several 256-row chunks and with mask pointers that are not 4-byte aligned.  Output buffers carry guard regions."""
import ctypes as C

import numpy as np
import pytest

import es_ref as R

pytestmark = pytest.mark.gpu

GUARD = 300


@pytest.fixture(scope="module")
def lib():
    import torch
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    from paddlerobotics_b200 import _lib
    return _lib.load()


def _stream():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


class RingModel:
    """Sequential `x[mask]` appends into a ring of the same capacity, in torch."""

    def __init__(self, cap, od, ad, device):
        import torch
        self.cap, self.pos, self.size = cap, 0, 0
        self.data = [torch.zeros(cap, od, device=device), torch.zeros(cap, ad, device=device), torch.zeros(cap, device=device),
                     torch.zeros(cap, od, device=device), torch.zeros(cap, device=device)]

    def append(self, rows, mask=None):
        import torch
        rows = rows if mask is None else [x[mask.bool()] for x in rows]
        m = rows[0].shape[0]
        slots = (self.pos + torch.arange(m, device=rows[0].device)) % self.cap
        for d, x in zip(self.data, rows):
            d[slots] = x
        self.pos, self.size = (self.pos + m) % self.cap, min(self.size + m, self.cap)


class Out:
    """Five float32 sample outputs [batch, od], [batch, ad], [batch], [batch, od], [batch], each followed by GUARD NaNs."""

    def __init__(self, batch, od, ad):
        import torch
        shapes = [(batch, od), (batch, ad), (batch,), (batch, od), (batch,)]
        self.bufs = [torch.full((int(np.prod(s)) + GUARD,), float("nan"), device="cuda") for s in shapes]
        self.t = [b[:int(np.prod(s))].view(s) for b, s in zip(self.bufs, shapes)]

    def ptrs(self):
        return [x.data_ptr() for x in self.t]

    def check(self):
        for b, x in zip(self.bufs, self.t):
            assert b[x.numel():].isnan().all(), "write past the end of a sample output"


def _rows(n, od, ad, g):
    import torch
    return [torch.randn(n, od, device="cuda", generator=g), torch.rand(n, ad, device="cuda", generator=g) * 2 - 1, torch.randn(n, device="cuda", generator=g),
            torch.randn(n, od, device="cuda", generator=g), (torch.rand(n, device="cuda", generator=g) > 0.1).float()]


class Ring:
    """Ring storage with a guard row block after each array (filled with NaN), and a guarded device cursor."""

    def __init__(self, cap, od, ad):
        import torch
        self.cap, self.od, self.ad = cap, od, ad
        shapes = [(cap, od), (cap, ad), (cap,), (cap, od), (cap,)]
        self.bufs = [torch.full((int(np.prod(s)) + GUARD,), float("nan"), device="cuda") for s in shapes]
        self.t = [b[:int(np.prod(s))].view(s) for b, s in zip(self.bufs, shapes)]
        for x in self.t:
            x.zero_()
        self.cur_buf = torch.full((3 + 8,), -77, dtype=torch.int64, device="cuda")
        self.cursor = self.cur_buf[:3]
        self.cursor.zero_()

    def ptrs(self):
        return [x.data_ptr() for x in self.t]

    def check(self):
        for b, x in zip(self.bufs, self.t):
            assert b[x.numel():].isnan().all(), "write past the end of the ring"
        assert (self.cur_buf[3:] == -77).all()

    def append(self, lib, rows, pos):
        assert lib.b2q_rpm_append(*self.ptrs(), *[x.data_ptr() for x in rows], None, rows[0].shape[0], self.od, self.ad, pos, self.cap, _stream()) == 0

    def append_cursor(self, lib, rows):
        assert lib.b2q_rpm_append_cursor(*self.ptrs(), *[x.data_ptr() for x in rows], rows[0].shape[0], self.od, self.ad, self.cap, self.cursor.data_ptr(),
                                         _stream()) == 0

    def append_masked(self, lib, rows, mask_ptr, n):
        assert lib.b2q_rpm_append_masked_cursor(*self.ptrs(), *[x.data_ptr() for x in rows], mask_ptr, n, self.od, self.ad, self.cap,
                                                self.cursor.data_ptr(), _stream()) == 0

    def sample(self, lib, batch, size, seed):
        out = Out(batch, self.od, self.ad)
        assert lib.b2q_rpm_sample(*self.ptrs(), *out.ptrs(), batch, self.od, self.ad, size, C.c_uint64(seed), _stream()) == 0
        out.check()
        return out.t

    def sample_cursor(self, lib, batch, seed):
        out = Out(batch, self.od, self.ad)
        assert lib.b2q_rpm_sample_cursor(*self.ptrs(), *out.ptrs(), batch, self.od, self.ad, C.c_uint64(seed), self.cursor.data_ptr(), _stream()) == 0
        out.check()
        return out.t


def _assert_gathered(got, ring, slots):
    """Every output row equals the ring row at the reference slot, bit for bit."""
    import torch
    idx = torch.as_tensor(slots, device="cuda")
    for g, r in zip(got, ring):
        want = r[idx]
        assert torch.equal(g.view(torch.int32), want.view(torch.int32)), "sampled rows differ from ring[slot]"


def _assert_ring(ring, model):
    import torch
    for got, want in zip(ring.t, model.data):
        assert torch.equal(got, want)


# ---- sampling
@pytest.mark.parametrize("size", [1, 2, 3, 1000, 2 ** 20 + 7])
def test_sample_gathers_exactly_the_reference_slots(lib, size):
    """b2q_rpm_sample and b2q_rpm_sample_cursor for batch 1, 64 and 8193, against rpm_slots: the plain call keys by `seed`, the cursor call
    by seed + state[2] and then increments state[2].  The ring is larger than `size` and its rows beyond `size` are never drawn."""
    import torch
    od, ad = 49, 12
    cap = size + 5
    ring = Ring(cap, od, ad)
    g = torch.Generator(device="cuda"); g.manual_seed(size)
    for x, y in zip(ring.t, _rows(cap, od, ad, g)):
        x.copy_(y)
    ring.cursor.copy_(torch.tensor([3, size, 41], device="cuda"))
    for batch in (1, 64, 8193):
        for seed in (0, 5, 2 ** 63 + 12345):
            got = ring.sample(lib, batch, size, seed)
            slots = R.rpm_slots(seed, batch, size)
            assert slots.max() < size
            _assert_gathered(got, ring.t, slots)
            count = int(ring.cursor[2])
            got = ring.sample_cursor(lib, batch, seed)
            _assert_gathered(got, ring.t, R.rpm_slots((seed + count) % 2 ** 64, batch, size))
            assert ring.cursor.tolist() == [3, size, count + 1]
    ring.check()


def test_replay_memory_seed_conventions(lib):
    """ReplayMemory.sample_batch: in host-cursor mode with seed=None the key is the sample count after this call's increment (1 for the
    first call); with a seed it is that seed.  In device-cursor mode the key is seed + state[2] (seed=None: 0 + state[2]), and the count
    increments after the draw."""
    import torch
    from paddlerobotics_b200.replay import ReplayMemory
    od, ad, n = 46, 12, 700
    g = torch.Generator(device="cuda"); g.manual_seed(3)
    rows = _rows(n, od, ad, g)
    host, dev = ReplayMemory(1000, od, ad), ReplayMemory(1000, od, ad, device_cursor=True)
    host.append(*rows); dev.append(*rows)
    ring = [host.obs, host.action, host.reward, host.next_obs, host.terminal]
    for k in range(3):
        _assert_gathered(host.sample_batch(257), ring, R.rpm_slots(k + 1, 257, n))
    _assert_gathered(host.sample_batch(64, seed=9), ring, R.rpm_slots(9, 64, n))
    assert host._samples == 4
    for k in range(3):
        _assert_gathered(dev.sample_batch(257), ring, R.rpm_slots(k, 257, n))
    _assert_gathered(dev.sample_batch(64, seed=9), ring, R.rpm_slots(9 + 3, 64, n))
    assert dev.cursor.tolist() == [n, n, 4] and dev._samples == 4


def test_sample_after_partial_masked_appends_draws_only_filled_slots(lib):
    """Masked appends that leave the ring partly filled: the device-cursor sample draws from [0, state[1]) only."""
    import torch
    od, ad, n, cap = 49, 12, 500, 4000
    ring = Ring(cap, od, ad)
    model = RingModel(cap, od, ad, "cuda")
    g = torch.Generator(device="cuda"); g.manual_seed(8)
    for k in range(3):
        rows = _rows(n, od, ad, g)
        mask = (torch.rand(n, device="cuda", generator=g) < 0.4).to(torch.uint8)
        ring.append_masked(lib, rows, mask.data_ptr(), n)
        model.append(rows, mask)
    size = model.size
    assert 0 < size < cap and ring.cursor.tolist() == [size, size, 0]
    for batch in (1, 64, 8193):
        got = ring.sample_cursor(lib, batch, 17)
        slots = R.rpm_slots(17 + int(ring.cursor[2]) - 1, batch, size)
        _assert_gathered(got, ring.t, slots)
        assert not got[0].isnan().any() and (got[0].abs().sum(1) > 0).all()     # no empty (zero) slot beyond the fill level is drawn
    _assert_ring(ring, model)
    ring.check()


# ---- appends at every row width
@pytest.mark.parametrize("od", [1, 46, 49, 64, 65, 294])
@pytest.mark.parametrize("ad", [1, 12, 60])
def test_appends_and_samples_at_row_widths(lib, od, ad):
    """Plain (host position), cursor and masked appends that wrap the ring, each against the torch ring model, then both samplers; the
    widths straddle the 64-thread stride of the plain and cursor kernels and the 32-lane stride of the masked kernel (60: the HYBRID
    action, 294: a 6 x 49 stacked history)."""
    import torch
    cap, n = 333, 150
    g = torch.Generator(device="cuda"); g.manual_seed(od * 100 + ad)
    plain, cur = Ring(cap, od, ad), Ring(cap, od, ad)
    mp, mc = RingModel(cap, od, ad, "cuda"), RingModel(cap, od, ad, "cuda")
    for k in range(4):                                                       # 600 rows: wraps
        rows = _rows(n, od, ad, g)
        plain.append(lib, rows, mp.pos); mp.append(rows)
        if k % 2:
            mask = (torch.rand(n, device="cuda", generator=g) < 0.6).to(torch.uint8) * 3
            cur.append_masked(lib, rows, mask.data_ptr(), n); mc.append(rows, mask)
        else:
            cur.append_cursor(lib, rows); mc.append(rows)
    _assert_ring(plain, mp)
    _assert_ring(cur, mc)
    assert cur.cursor.tolist() == [mc.pos, mc.size, 0]
    _assert_gathered(plain.sample(lib, 129, mp.size, 4), plain.t, R.rpm_slots(4, 129, mp.size))
    _assert_gathered(cur.sample_cursor(lib, 129, 4), cur.t, R.rpm_slots(4, 129, mc.size))
    plain.check(); cur.check()


# ---- masked append at large n
@pytest.mark.parametrize("n", [16385, 131073, 300000])
def test_masked_append_large_n(lib, n):
    """n = 16385, 131073 and 300000 give tiles of 64, 288 and 608 rows: one, two and three 256-row chunks per CTA.  cap == n; masks with
    only the first row valid, only the last, random density 0.3, and all rows; the appends wrap the ring."""
    import torch
    od, ad = 49, 12
    ring = Ring(n, od, ad)
    model = RingModel(n, od, ad, "cuda")
    g = torch.Generator(device="cuda"); g.manual_seed(n)
    masks = []
    m = torch.zeros(n, dtype=torch.uint8, device="cuda"); m[0] = 1; masks.append(m)
    m = torch.zeros(n, dtype=torch.uint8, device="cuda"); m[-1] = 255; masks.append(m)
    masks.append((torch.rand(n, device="cuda", generator=g) < 0.3).to(torch.uint8))
    masks.append(torch.ones(n, dtype=torch.uint8, device="cuda"))
    masks.append((torch.rand(n, device="cuda", generator=g) < 0.3).to(torch.uint8))
    for mask in masks:
        rows = _rows(n, od, ad, g)
        ring.append_masked(lib, rows, mask.data_ptr(), n)
        model.append(rows, mask)
        assert ring.cursor.tolist() == [model.pos, model.size, 0]
    _assert_ring(ring, model)
    ring.check()


@pytest.mark.parametrize("offset", [1, 2, 3])
def test_masked_append_misaligned_mask(lib, offset):
    """Mask pointers 1, 2 and 3 bytes into a larger buffer (count_valid's byte-wise head), through the C call at several sizes and through
    ReplayMemory.append_masked with a sliced uint8 view (.contiguous() keeps the offset)."""
    import torch
    from paddlerobotics_b200.replay import ReplayMemory
    od, ad = 49, 12
    for n in (1, 2, 3, 5, 1000, 131073):
        ring = Ring(n, od, ad)
        model = RingModel(n, od, ad, "cuda")
        g = torch.Generator(device="cuda"); g.manual_seed(n * 4 + offset)
        buf = torch.full((n + 8,), 1, dtype=torch.uint8, device="cuda")     # the bytes around the mask are valid: reading them would count
        for density in (0.5, 0.05):
            mask = buf[offset:offset + n]
            mask.copy_((torch.rand(n, device="cuda", generator=g) < density).to(torch.uint8))
            mask[0] = 1 if density > 0.1 else 0
            assert mask.data_ptr() % 4 == offset % 4
            rows = _rows(n, od, ad, g)
            ring.append_masked(lib, rows, mask.data_ptr(), n)
            model.append(rows, mask)
            assert ring.cursor.tolist() == [model.pos, model.size, 0]
        _assert_ring(ring, model)
        ring.check()
    n = 4097
    g = torch.Generator(device="cuda"); g.manual_seed(offset)
    for device_cursor in (False, True):
        rpm = ReplayMemory(5000, od, ad, device_cursor=device_cursor)
        model = RingModel(5000, od, ad, "cuda")
        buf = torch.ones(n + 8, dtype=torch.uint8, device="cuda")
        for k in range(3):
            view = buf[offset:offset + n]
            view.copy_((torch.rand(n, device="cuda", generator=g) < 0.4).to(torch.uint8))
            assert view.contiguous().data_ptr() % 4 == offset % 4
            rows = _rows(n, od, ad, g)
            rpm.append_masked(*rows, view)
            model.append(rows, view)
        for got, want in zip([rpm.obs, rpm.action, rpm.reward, rpm.next_obs, rpm.terminal], model.data):
            assert torch.equal(got, want)
        assert rpm.size() == model.size and (rpm._curr_pos, rpm._curr_size) == (model.pos, model.size)
