"""GPU parity tests for EXE (EXECodec, transform/EXECodec.go) and for the complete chain of kanzi -l 4
(TEXT+UTF+EXE+PACK+MM+ROLZ & NONE). The per-block logic is kz_exe_core.cuh, checked on the CPU by tests/test_exe_core_host.py."""
import sys

import numpy as np
import pytest

from test_oracle_pre import _synth_arm64, _synth_x86

pytestmark = pytest.mark.gpu

T_EXE = 9


def cases(synth, n, seed):
    yield "x86", _synth_x86(n, seed)
    yield "arm64", _synth_arm64(n, seed + 1)
    yield "uniform", synth.uniform_bytes(n, seed=seed + 2)
    yield "text", synth.markov_text(n, seed=seed + 3)
    exe = np.fromfile(sys.executable, dtype=np.uint8)
    if len(exe) >= n and bytes(exe[:4]) == b"\x7fELF":
        yield "elf", exe[:n].copy()
        yield "elf_tail", exe[len(exe) - n:].copy()


@pytest.mark.parametrize("n", [4000, 4096, 100003, 1 << 20])
def test_exe_transform_parity(gpu, oracle, synth, kz, n):
    for cname, x in cases(synth, n, seed=n):
        for dt in (0, 3, 7, 1):
            want, wdt = oracle.transform_forward(T_EXE, x, dt)
            got, gdt = gpu.transform_forward(T_EXE, x, dt)
            assert gdt == wdt, (cname, n, dt, gdt, wdt)
            if want is None:
                assert got is None, (cname, n, dt)
                continue
            assert got is not None, (cname, n, dt)
            m = min(len(got), len(want))
            assert len(got) == len(want) and np.array_equal(got, want), (cname, n, dt, len(got), len(want), int(np.argmax(got[:m] != want[:m])))
            back = gpu.transform_inverse(T_EXE, want, n + 64)
            assert np.array_equal(back, x), (cname, n, dt)


def test_exe_malformed_headers_behave_like_the_oracle(gpu, oracle, synth, kz):
    """header fields pointing outside the block: where the reference indexes out of bounds (a panic, i.e. a block error) the GPU reports an
    error too; where it reads garbage and carries on, the GPU produces the same bytes"""
    exe = np.fromfile(sys.executable, dtype=np.uint8)
    if len(exe) < (1 << 20) or bytes(exe[:4]) != b"\x7fELF":
        pytest.skip("no ELF interpreter to borrow a header from")
    variants = []
    for lo, hi, val in [(0x28, 0x30, 0xFF), (0x3C, 0x3E, 0xFF), (0x28, 0x30, 0x7F), (0x3A, 0x3C, 0xFF), (0x28, 0x2C, 0xF0)]:
        bad = exe[: 1 << 20].copy()
        bad[lo:hi] = val
        variants.append(bad)
    neg = exe[: 1 << 20].copy()
    neg[0x28:0x30] = [0x9C, 0xFF, 0xFF, 0xFF, 0xFF, 0xFF, 0xFF, 0xFF]  # section table at offset -100: a negative slice index panics
    variants.append(neg)
    mz = _synth_x86(1 << 16, 5).copy()
    mz[:2] = [0x4D, 0x5A]
    mz[60:64] = [0xF0, 0xFF, 0, 0]  # PE header offset near the end of the block
    variants.append(mz)
    macho = _synth_x86(1 << 16, 6).copy()
    macho[:4] = [0xCF, 0xFA, 0xED, 0xFE]
    macho[12:16] = [2, 0, 0, 0]
    macho[16:20] = [40, 0, 0, 0]  # 40 load commands of random sizes
    variants.append(macho)
    for i, bad in enumerate(variants):
        try:
            want, wdt = oracle.transform_forward(T_EXE, bad)
        except oracle.OracleError:
            with pytest.raises(kz.KanziError):
                gpu.transform_forward(T_EXE, bad)
            continue
        got, gdt = gpu.transform_forward(T_EXE, bad)
        assert (want is None) == (got is None) and gdt == wdt, i
        if want is not None:
            assert np.array_equal(got, want), i


@pytest.mark.parametrize("bs", [8192, 1 << 17])
def test_stream_parity_level4_chain(gpu, oracle, synth, kz, bs):
    """kanzi -l 4 = TEXT+UTF+EXE+PACK+MM+ROLZ & NONE: six transforms, every one on the GPU"""
    r = np.random.default_rng(bs)
    t = np.arange(bs)
    wave = (128 + 100 * np.sin(t / 40.0) + r.normal(0, 1.5, bs)).astype(np.uint8)
    parts = [synth.markov_text(bs, seed=bs), _synth_x86(bs, bs + 1), wave, synth.uniform_bytes(bs, seed=bs + 2), _synth_arm64(bs, bs + 3),
             np.frombuffer(b"ACGT", np.uint8)[synth.uniform_bytes(bs, seed=bs + 4) & 3], _synth_x86(bs // 2 + 9, bs + 5)]
    exe = np.fromfile(sys.executable, dtype=np.uint8)
    if len(exe) >= 3 * bs:
        parts.insert(1, exe[: 3 * bs].copy())  # first block starts with the ELF magic: data type EXE from the start
    x = np.concatenate(parts)
    n = len(x)
    want = oracle.compress(x, "TEXT+UTF+EXE+PACK+MM+ROLZ", "NONE", block_size=bs, jobs=8, input_size=n)
    got = gpu.compress(x, "TEXT+UTF+EXE+PACK+MM+ROLZ", "NONE", block_size=bs, input_size=n)
    m = min(len(got), len(want))
    assert len(got) == len(want) and np.array_equal(got, want), (bs, len(got), len(want), int(np.argmax(got[:m] != want[:m])))
    assert np.array_equal(gpu.decompress(want, n + 64), x), bs


@pytest.mark.parametrize("n,seed", [(4096, 1), (65536, 3), (1 << 20, 5)])
def test_exe_x86_blocks_of_the_independent_pin(gpu, oracle, kz, n, seed):
    """the blocks tests/test_oracle_exe_independent.py pins the oracle with (a third, Python statement of EXECodec.go's x86 path): GPU == that statement"""
    from test_oracle_exe_independent import forward_x86, make_block

    x = make_block(n, seed)
    want = forward_x86(x)
    got, _ = gpu.transform_forward(kz.TRANSFORM_IDS["EXE"], x)
    assert want is not None and got is not None and len(got) == len(want) and np.array_equal(got, want)
    back = gpu.transform_inverse(kz.TRANSFORM_IDS["EXE"], want, n + 64)
    assert np.array_equal(back, x)


@pytest.mark.parametrize("n,seed", [(4096, 21), (300004, 23)])
def test_exe_arm64_blocks_of_the_independent_pin(gpu, oracle, kz, n, seed):
    from test_oracle_exe_independent import forward_arm, make_arm_block

    x = make_arm_block(n, seed)
    want = forward_arm(x)
    got, _ = gpu.transform_forward(kz.TRANSFORM_IDS["EXE"], x)
    assert want is not None and got is not None and len(got) == len(want) and np.array_equal(got, want)
    back = gpu.transform_inverse(kz.TRANSFORM_IDS["EXE"], want, n + 64)
    assert np.array_equal(back, x)
