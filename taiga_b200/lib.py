"""ctypes binding of libtaiga_b200.so (C ABI declared in include/taiga_b200.h).

The product path has no CPU fallback: if the CUDA library is missing or no sm_90 device is usable this
module raises instead of computing anything on the host.
"""
import collections
import ctypes
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libtaiga_b200.so")

TB_FP, TB_FQ = 0, 1
TB_VESTA, TB_PALLAS = 0, 1
TB_OK, TB_ERR_INVALID, TB_ERR_CUDA, TB_ERR_CONSTRAINT, TB_ERR_INTERNAL = 0, 1, 2, 3, 4
# status of one proof of tb_dev_prove_batch: proved, 1 + l (an input of lookup l is not in its table), or an internal error
# (0xFFFFFFFF, which reads as -1 in the int32 status tensors of ProvingKey.prove_batch_dev)
TB_PROVED, TB_PROVE_INTERNAL = 0, 0xFFFFFFFF


class TaigaB200Error(RuntimeError):
    def __init__(self, status, msg):
        super().__init__("libtaiga_b200 status %d: %s" % (status, msg))
        self.status = status


class ConstraintSystemFailure(TaigaB200Error):
    """Mirror of halo2 `plonk::Error::ConstraintSystemFailure` (the witness does not satisfy the circuit)."""


_lib = None
_vp, _sz, _u32, _i, _u64 = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_uint32, ctypes.c_int, ctypes.c_uint64

_SIGS = {
    "tb_ctx_create": (_i, [_i, ctypes.POINTER(_vp)]),
    "tb_ctx_destroy": (None, [_vp]),
    "tb_last_error": (ctypes.c_char_p, [_vp]),
    "tb_version": (ctypes.c_char_p, []),
    "tb_ctx_sync": (_i, [_vp]),
    "tb_ctx_stream": (_u64, [_vp]),
    "tb_ctx_launch_count": (_u64, [_vp]),
    "tb_prof_categories": (_i, []),
    "tb_prof_category_name": (ctypes.c_char_p, [_i]),
    "tb_prof_enable": (_i, [_vp, _i]),
    "tb_prof_read": (_i, [_vp, _vp, _vp]),
    "tb_prof_work": (_i, [_vp, _vp]),
    "tb_ntt": (_i, [_vp, _i, _u32, _i, _i, _u32, _vp, _vp]),
    "tb_msm": (_i, [_vp, _i, _sz, _u32, _vp, _vp, _u32, _vp]),
    "tb_dev_to_mont": (_i, [_vp, _i, _vp, _sz]),
    "tb_dev_from_mont": (_i, [_vp, _i, _vp, _sz]),
    "tb_dev_ntt": (_i, [_vp, _i, _u32, _i, _i, _u32, _vp, _vp, _vp]),
    "tb_dev_msm": (_i, [_vp, _i, _sz, _u32, _vp, _vp, _u32, _vp]),
    "tb_dev_verify_batch_vk": (_i, [_vp, _vp, _u32, _vp, _vp, _vp, _sz, _sz, _vp]),
    "tb_dev_batch_verifier_add": (_i, [_vp, _vp, _vp, _u32, _vp, _vp, _vp, _sz, _sz]),
    "tb_srs_load": (_i, [_vp, _u32, _vp, _vp, _vp, _vp, ctypes.POINTER(_vp)]),
    "tb_srs_free": (None, [_vp]),
    "tb_srs_commit": (_i, [_vp, _vp, _i, _u32, _vp, _vp, _vp]),
    "tb_circuit_load": (_i, [_vp, _vp, _vp, _vp, _vp, ctypes.POINTER(_vp)]),
    "tb_pk_free": (None, [_vp]),
    "tb_pk_proof_len": (_sz, [_vp]),
    "tb_pk_commitments": (_i, [_vp, _vp, _vp, _vp]),
    "tb_prove_batch": (_i, [_vp, _vp, _u32, _vp, _vp, _vp, _vp, _u32, _vp, _sz]),
    "tb_dev_prove_batch": (_i, [_vp, _vp, _u32, _vp, _vp, _vp, _vp, _u32, _vp, _sz, _vp]),
    "tb_verify_batch": (_i, [_vp, _vp, _u32, _vp, _vp, _vp, _sz, _sz, _vp]),
    "tb_decompress": (_i, [_vp, _sz, _vp, _vp, _vp]),
    "tb_vk_load": (_i, [_vp, _vp, _vp, _vp, _vp, ctypes.POINTER(_vp)]),
    "tb_vk_free": (None, [_vp]),
    "tb_vk_proof_len": (_sz, [_vp]),
    "tb_verify_batch_vk": (_i, [_vp, _vp, _u32, _vp, _vp, _vp, _sz, _sz, _vp]),
    "tb_check_batch": (_i, [_vp, _vp, _u32, _vp, _vp, _vp, _vp, _u32, _vp, _vp]),
    "tb_batch_verifier_create": (_i, [_vp, _vp, _vp, ctypes.POINTER(_vp)]),
    "tb_batch_verifier_add": (_i, [_vp, _vp, _vp, _u32, _vp, _vp, _vp, _sz, _sz]),
    "tb_batch_verifier_finalize": (_i, [_vp, _vp, _vp]),
    "tb_batch_verifier_free": (None, [_vp]),
}

TB_FAIL_GATE, TB_FAIL_LOOKUP, TB_FAIL_COPY = 1, 2, 3
# one record of tb_check_batch (tb_failure): kind TB_FAIL_*; gate: constraint `index` on `row`; lookup: lookup `index`, input row
# `row`; copy: permutation column position `index`, `row`, and its sigma-successor (other_column, other_row)
Failure = collections.namedtuple("Failure", "kind index row other_column other_row")


def render_failure(keydata, f):
    """The message circuits_random.satisfied gives for failure `f` of a witness of `keydata`'s circuit."""
    cs = keydata.cs
    if f.kind == TB_FAIL_GATE:
        names = [(name, i) for name, polys in cs.gates for i in range(len(polys))]
        name, i = names[f.index]
        return "gate %s poly %d is not zero on row %d" % (name, i, f.row)
    if f.kind == TB_FAIL_LOOKUP:
        return "lookup %d: input on row %d is not in the table" % (f.index, f.row)
    if f.kind == TB_FAIL_COPY:
        cols = cs.perm_columns
        return "copy (%r, %d) -> (%r, %d) joins different values" % (cols[f.index], f.row, cols[f.other_column], f.other_row)
    raise ValueError("unknown failure kind %d" % f.kind)


def exported_symbols():
    """Every symbol include/taiga_b200.h declares (checked by the CPU test-suite)."""
    return sorted(_SIGS)


def load():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError("libtaiga_b200.so is not built (run `python -c 'import __graft_entry__ as g; g.build()'`); "
                              "there is no CPU fallback for the prover path")
        lib = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in _SIGS.items():
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = res, args
        _lib = lib
    return _lib


def _ptr(a):
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        assert a.flags["C_CONTIGUOUS"]
        return a.ctypes.data_as(_vp)
    if hasattr(a, "data_ptr"):  # torch tensor
        return _vp(a.data_ptr())
    return _vp(int(a))


def _u8(a):
    return np.ascontiguousarray(a, dtype=np.uint8)


class Context:
    """One GPU, one stream (tb_ctx)."""

    def __init__(self, device=0):
        self._lib = load()
        h = _vp()
        st = self._lib.tb_ctx_create(int(device), ctypes.byref(h))
        if st != TB_OK:
            raise TaigaB200Error(st, "tb_ctx_create failed: no usable sm_90 (H100) CUDA device (no CPU fallback exists)")
        self._h = h
        self.device = device

    def close(self):
        if getattr(self, "_h", None):
            self._lib.tb_ctx_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, st):
        if st != TB_OK:
            msg = self._lib.tb_last_error(self._h).decode(errors="replace")
            raise (ConstraintSystemFailure if st == TB_ERR_CONSTRAINT else TaigaB200Error)(st, msg)

    @property
    def stream(self):
        return int(self._lib.tb_ctx_stream(self._h))

    @property
    def launch_count(self):
        return int(self._lib.tb_ctx_launch_count(self._h))

    def sync(self):
        self._check(self._lib.tb_ctx_sync(self._h))

    def prof_enable(self, on=True):
        self._check(self._lib.tb_prof_enable(self._h, int(on)))

    def prof_read(self):
        """{category: (milliseconds, kernel groups)} since the last read, measured with CUDA events on the context's stream."""
        n = self._lib.tb_prof_categories()
        ms = np.zeros(n, np.float64)
        cnt = np.zeros(n, np.uint64)
        self._check(self._lib.tb_prof_read(self._h, _ptr(ms), _ptr(cnt)))
        return {self._lib.tb_prof_category_name(i).decode(): (float(ms[i]), int(cnt[i])) for i in range(n)}

    def work_read(self):
        """{category: Montgomery multiplications executed since the last read} (the numerator of the integer-pipe roofline)."""
        n = self._lib.tb_prof_categories()
        mm = np.zeros(n, np.float64)
        self._check(self._lib.tb_prof_work(self._h, _ptr(mm)))
        return {self._lib.tb_prof_category_name(i).decode(): float(mm[i]) for i in range(n)}

    # ---- host-buffer primitives
    def ntt(self, field, data, inverse=False, coset=False, batch=1):
        d = _u8(data)
        n = d.size // 32 // batch
        logn = n.bit_length() - 1
        assert (1 << logn) == n and d.size == batch * n * 32
        out = np.empty_like(d)
        self._check(self._lib.tb_ntt(self._h, field, logn, int(inverse), int(coset), batch, _ptr(d), _ptr(out)))
        return out.reshape(batch * n, 32) if batch > 1 else out.reshape(n, 32)

    def msm(self, curve, scalars, points, batch=1, window_bits=0):
        s, p = _u8(scalars), _u8(points)
        n = p.size // 64
        assert s.size == batch * n * 32
        out = np.zeros((batch, 64), np.uint8)
        self._check(self._lib.tb_msm(self._h, curve, n, batch, _ptr(s), _ptr(p), window_bits, _ptr(out)))
        return out

    def decompress(self, encodings):
        """Compressed Vesta points [n, 32] -> (affine points uint8 [n, 64], accepted bool [n]); a rejected encoding gives
        64 zero bytes, and so does the identity (32 zero bytes), which is accepted."""
        e = _u8(encodings).reshape(-1, 32)
        n = e.shape[0]
        out = np.zeros((n, 64), np.uint8)
        ok = np.zeros(n, np.uint8)
        self._check(self._lib.tb_decompress(self._h, n, _ptr(e), _ptr(out), _ptr(ok)))
        return out, ok.astype(bool)

    # ---- device-buffer primitives (torch tensors / raw device pointers)
    def dev_to_mont(self, field, t, n):
        self._check(self._lib.tb_dev_to_mont(self._h, field, _ptr(t), n))

    def dev_from_mont(self, field, t, n):
        self._check(self._lib.tb_dev_from_mont(self._h, field, _ptr(t), n))

    def dev_ntt(self, field, logn, d_in, d_out, d_scratch, inverse=False, coset=False, batch=1):
        self._check(self._lib.tb_dev_ntt(self._h, field, logn, int(inverse), int(coset), batch, _ptr(d_in), _ptr(d_out), _ptr(d_scratch)))

    def dev_msm(self, curve, n, d_scalars, d_points, d_out, batch=1, window_bits=0):
        self._check(self._lib.tb_dev_msm(self._h, curve, n, batch, _ptr(d_scalars), _ptr(d_points), window_bits, _ptr(d_out)))

    def load_srs(self, k, g, g_lagrange, w, u):
        return Srs(self, k, g, g_lagrange, w, u)


class Srs:
    """Device-resident Params<vesta::Affine> (constant.rs:128-139) with fixed-base tables."""

    def __init__(self, ctx, k, g, g_lagrange, w, u):
        self.ctx, self.k, self.n = ctx, k, 1 << k
        g, gl, w, u = _u8(g), _u8(g_lagrange), _u8(w), _u8(u)
        assert g.size == 64 * self.n and gl.size == 64 * self.n and w.size == 64 and u.size == 64
        h = _vp()
        ctx._check(ctx._lib.tb_srs_load(ctx._h, k, _ptr(g), _ptr(gl), _ptr(w), _ptr(u), ctypes.byref(h)))
        self._h = h

    def commit(self, scalars, blinds=None, lagrange=False, batch=1):
        """Params::commit / commit_lagrange: MSM(scalars, g | g_lagrange) + blind * w, per batch item."""
        s = _u8(scalars)
        assert s.size == batch * self.n * 32
        b = _u8(blinds) if blinds is not None else None
        out = np.zeros((batch, 64), np.uint8)
        self.ctx._check(self.ctx._lib.tb_srs_commit(self.ctx._h, self._h, int(lagrange), batch, _ptr(s), _ptr(b), _ptr(out)))
        return out

    def load_circuit(self, keydata):
        return ProvingKey(self, keydata)

    def load_verifying_key(self, keydata, fixed, sigma):
        """VerifyingKey from the circuit description of `keydata` and the vk's commitments: fixed [num_fixed, 64],
        sigma [num_perm_columns, 64] (what ProvingKey.commitments() returns).  keydata.fixed / keydata.sigma are not read."""
        return VerifyingKey(self, keydata, fixed, sigma)

    def close(self):
        if getattr(self, "_h", None):
            self.ctx._lib.tb_srs_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class ProvingKey:
    """Device-resident proving key of one circuit (tb_pk): the stand-in for halo2's ProvingKey<vesta::Affine>
    (COMPLIANCE_PROVING_KEY / TRIVIAL_RESOURCE_LOGIC_PK, constant.rs:145-152, resource_logic_examples.rs:50-61).
    `keydata` is a taiga_b200.circuit.CircuitKeyData (descriptor + fixed columns + sigma)."""

    def __init__(self, srs, keydata):
        self.srs, self.ctx, self.keydata = srs, srs.ctx, keydata
        self._fixed, self._sigma = _u8(keydata.fixed), _u8(keydata.sigma)
        h = _vp()
        self.ctx._check(self.ctx._lib.tb_circuit_load(self.ctx._h, srs._h, ctypes.byref(keydata.desc), _ptr(self._fixed), _ptr(self._sigma), ctypes.byref(h)))
        self._h = h
        self.proof_len = int(self.ctx._lib.tb_pk_proof_len(h))

    def commitments(self):
        """keygen_vk: (fixed column commitments [num_fixed, 64], sigma commitments [P, 64])."""
        kd = self.keydata
        f = np.zeros((max(1, kd.cs.num_fixed), 64), np.uint8)
        s = np.zeros((max(1, len(kd.cs.perm_columns)), 64), np.uint8)
        self.ctx._check(self.ctx._lib.tb_pk_commitments(self.ctx._h, self._h, _ptr(f), _ptr(s)))
        return f[: kd.cs.num_fixed], s[: len(kd.cs.perm_columns)]

    def prove_batch(self, advice, instance, instance_len, seed, first_proof_index=0):
        """Proof::create for a batch: advice uint8 [B, num_advice, n, 32]; instance uint8 [B, sum(instance_len), 32].
        Returns a list of B proof byte strings."""
        adv = _u8(advice)
        kd = self.keydata
        per = kd.cs.num_advice * kd.n * 32
        assert adv.size % per == 0
        return self.prove_batch_raw(adv, adv.size // per, instance, instance_len, seed, first_proof_index)

    def prove_batch_raw(self, advice, B, instance, instance_len, seed, first_proof_index=0, ctx=None):
        """Same, with `advice` given as anything exposing its address (numpy array, pinned-host or DEVICE torch tensor).
        `ctx`: run on another Context (= another CUDA stream) of the same device, e.g. to overlap two circuits."""
        ctx = ctx or self.ctx
        inst = _u8(instance)
        lens = np.ascontiguousarray(instance_len, dtype=np.uint32)
        assert inst.size >= B * int(lens.sum()) * 32
        seed = _u8(np.frombuffer(bytes(seed), np.uint8))
        assert seed.size == 32
        out = np.zeros((B, self.proof_len), np.uint8)
        ctx._check(ctx._lib.tb_prove_batch(ctx._h, self._h, B, _ptr(advice), _ptr(inst), _ptr(lens), _ptr(seed), first_proof_index,
                                           _ptr(out), self.proof_len))
        return [out[b].tobytes() for b in range(B)]

    def prove_batch_dev(self, advice, instance, instance_len, seed, proofs, status, first_proof_index=0, ctx=None):
        """prove_batch into device memory, enqueued on the context's stream without waiting (tb_dev_prove_batch).  `advice` a
        contiguous CUDA uint8 tensor of B witnesses (B * num_advice * n * 32 bytes), `instance` a contiguous CUDA uint8 tensor of
        B * sum(instance_len) * 32 bytes (or None without instance columns), `proofs` a CUDA uint8 tensor [B, >= proof_len] (one
        record per row, any row stride), `status` a CUDA int32 tensor of B statuses: TB_PROVED, 1 + l for a missing input of
        lookup l, or TB_PROVE_INTERNAL (reads as -1).  A record whose status is not TB_PROVED is all zeros.  The context's
        stream first waits for torch's current stream, and the tensors are kept from reuse until it has run the call (torch
        records an event on the context's stream when it frees them: free them before closing the context)."""
        ctx = ctx or self.ctx
        kd = self.keydata
        assert advice.is_cuda and advice.dtype.itemsize == 1 and advice.is_contiguous()
        assert status.is_cuda and str(status.dtype) == "torch.int32" and status.is_contiguous() and status.numel() >= proofs.shape[0]
        B, inst, lens, addr, stride, plen = _dev_args(ctx, instance, instance_len, proofs, None, advice, status)
        assert plen >= self.proof_len and advice.numel() == B * kd.cs.num_advice * kd.n * 32
        seed = _u8(np.frombuffer(bytes(seed), np.uint8))
        assert seed.size == 32
        ctx._check(ctx._lib.tb_dev_prove_batch(ctx._h, self._h, B, _vp(advice.data_ptr()), inst, _ptr(lens), _ptr(seed), first_proof_index,
                                               addr, stride, _vp(status.data_ptr())))

    def verify_batch(self, instance, instance_len, proofs, ctx=None):
        """Proof::verify for a batch: proofs = list of byte strings; returns a list of booleans."""
        return _verify_batch(ctx or self.ctx, "tb_verify_batch", self._h, instance, instance_len, proofs)

    def check_batch(self, advice, instance, instance_len, seed, max_failures=16, ctx=None):
        """MockProver::run(k, circuit, instance).verify() for a batch, without proving: advice / instance as in prove_batch
        (advice may also be a pinned-host or device torch tensor).  `seed` (32 bytes) draws the random fold of the gates and
        the compression of the lookups; it must be unpredictable to whoever wrote the witnesses.  Returns per witness
        (counts, failures): counts = (rows with a failing constraint, failing lookup inputs, failing copy cells), failures
        = the first max_failures Failure records, gates by (row, constraint), then lookups, then copies.  A witness passes
        iff all counts are 0; render_failure names a record as circuits_random.satisfied does."""
        ctx = ctx or self.ctx
        kd = self.keydata
        per = kd.cs.num_advice * kd.n * 32
        if hasattr(advice, "data_ptr"):
            nbytes = advice.numel() * advice.element_size()
        else:
            advice = _u8(advice)
            nbytes = advice.size
        assert nbytes % per == 0
        B = nbytes // per
        inst = _u8(instance)
        lens = np.ascontiguousarray(instance_len, dtype=np.uint32)
        assert inst.size >= B * int(lens.sum()) * 32
        seed = _u8(np.frombuffer(bytes(seed), np.uint8))
        assert seed.size == 32
        counts = np.zeros((B, 3), np.uint64)
        recs = np.zeros((B, max(1, max_failures), 5), np.uint32)
        ctx._check(ctx._lib.tb_check_batch(ctx._h, self._h, B, _ptr(advice), _ptr(inst), _ptr(lens), _ptr(seed), max_failures,
                                           _ptr(counts), _ptr(recs) if max_failures else None))
        out = []
        for b in range(B):
            fails = [Failure(*(int(v) for v in r)) for r in recs[b, :max_failures] if r[0]]   # unused records are zero
            out.append((tuple(int(c) for c in counts[b]), fails))
        return out

    def verifying_key(self):
        """The VerifyingKey of this circuit, built from commitments(): it holds no device table and verifies without this key."""
        f, s = self.commitments()
        return VerifyingKey(self.srs, self.keydata, f, s)

    def close(self):
        if getattr(self, "_h", None):
            self.ctx._lib.tb_pk_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _host_args(instance, instance_len, proofs):
    """(n_proofs, instance, instance_len, proofs, proof_stride, proof_len) of a verifier call on host memory: `proofs` byte
    strings of one length, packed one after the other."""
    B = len(proofs)
    plen = len(proofs[0]) if B else 0
    assert all(len(p) == plen for p in proofs)
    buf = np.frombuffer(b"".join(proofs), np.uint8).copy() if B else np.zeros(1, np.uint8)
    return B, _u8(instance), np.ascontiguousarray(instance_len, dtype=np.uint32), buf, plen, plen


def _verify_batch(ctx, fn, h, instance, instance_len, proofs):
    B, inst, lens, buf, stride, plen = _host_args(instance, instance_len, proofs)
    ok = np.zeros(B, np.uint8)
    ctx._check(getattr(ctx._lib, fn)(ctx._h, h, B, _ptr(inst), _ptr(lens), _ptr(buf), stride, plen, _ptr(ok)))
    return [bool(v) for v in ok]


def _dev_args(ctx, instance, instance_len, proofs, proof_len, *tensors):
    """(n_proofs, instance, instance_len, proofs, proof_stride, proof_len) of a prover or verifier call on device memory:
    `proofs` a CUDA uint8 tensor of B proof records, one per row (rows may be padded or be views with any row stride;
    proof_len defaults to the row length), read by the verifier and written by the prover; `instance` a contiguous CUDA uint8
    tensor or None; `tensors` the call's other device buffers (verdicts; advice and statuses).  Orders the context's stream
    after the work torch has enqueued on its current stream (what made or last read the tensors), and marks `proofs`,
    `instance` and `tensors` as used on the context's stream, so that torch's allocator does not hand their memory out again
    before the call has run there."""
    import torch
    assert proofs.is_cuda and proofs.dtype.itemsize == 1 and proofs.dim() == 2 and proofs.stride(1) == 1
    assert instance is None or (instance.is_cuda and instance.dtype.itemsize == 1 and instance.is_contiguous())
    dev = proofs.device
    s = torch.cuda.ExternalStream(ctx.stream, device=dev)
    ev = torch.cuda.Event()
    ev.record(torch.cuda.current_stream(dev))
    s.wait_event(ev)
    for t in (proofs, instance) + tensors:
        if t is not None:
            t.record_stream(s)
    inst = None if instance is None or instance.numel() == 0 else _vp(instance.data_ptr())
    return (proofs.shape[0], inst, np.ascontiguousarray(instance_len, dtype=np.uint32), _vp(proofs.data_ptr()), proofs.stride(0),
            proofs.shape[1] if proof_len is None else int(proof_len))


class VerifyingKey:
    """The verifying key of one circuit (tb_vk): halo2's VerifyingKey<vesta::Affine> as Proof::verify uses it
    (proof.rs:45-54).  Holds the circuit's shape and the fixed / sigma commitments in host memory; refers to `srs`."""

    def __init__(self, srs, keydata, fixed, sigma):
        self.srs, self.ctx = srs, srs.ctx
        cs = keydata.cs
        f, s = _u8(fixed).reshape(-1, 64), _u8(sigma).reshape(-1, 64)
        assert f.shape[0] == cs.num_fixed and s.shape[0] == len(cs.perm_columns)
        f, s = np.ascontiguousarray(f), np.ascontiguousarray(s)
        h = _vp()
        self.ctx._check(self.ctx._lib.tb_vk_load(self.ctx._h, srs._h, ctypes.byref(keydata.desc), _ptr(f) if f.size else None,
                                                 _ptr(s) if s.size else None, ctypes.byref(h)))
        self._h = h
        self.proof_len = int(self.ctx._lib.tb_vk_proof_len(h))

    def verify_batch(self, instance, instance_len, proofs, ctx=None):
        """Proof::verify for a batch: proofs = list of byte strings; returns a list of booleans."""
        return _verify_batch(ctx or self.ctx, "tb_verify_batch_vk", self._h, instance, instance_len, proofs)

    def verify_batch_dev(self, instance, instance_len, proofs, ok, ctx=None, proof_len=None):
        """verify_batch over device memory, enqueued on the context's stream without waiting (tb_dev_verify_batch_vk):
        `proofs` a CUDA uint8 tensor [B, >= proof_len] (one proof per row, any row stride), `instance` a contiguous CUDA
        uint8 tensor of B * sum(instance_len) * 32 bytes, `ok` a CUDA uint8 tensor of B verdicts written in stream order.  The
        context's stream first waits for torch's current stream, and the tensors are kept from reuse until it has run the call."""
        ctx = ctx or self.ctx
        assert ok.is_cuda and ok.dtype.itemsize == 1 and ok.is_contiguous() and ok.numel() >= proofs.shape[0]
        B, inst, lens, addr, stride, plen = _dev_args(ctx, instance, instance_len, proofs, proof_len, ok)
        ctx._check(ctx._lib.tb_dev_verify_batch_vk(ctx._h, self._h, B, inst, _ptr(lens), addr, stride, plen, _vp(ok.data_ptr())))

    def close(self):
        if getattr(self, "_h", None):
            self.ctx._lib.tb_vk_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class BatchVerifier:
    """halo2's plonk::BatchVerifier over the device (tb_batch_verifier): proofs of any circuits whose verifying keys refer to
    `srs`, added in any number of calls, then one verdict from finalize().  `seed` (32 bytes) draws the proofs' random weights;
    it must be unpredictable to whoever made the proofs: draw a fresh one per batch."""

    def __init__(self, srs, seed):
        self.srs, self.ctx = srs, srs.ctx
        seed = _u8(np.frombuffer(bytes(seed), np.uint8))
        assert seed.size == 32
        h = _vp()
        self.ctx._check(self.ctx._lib.tb_batch_verifier_create(self.ctx._h, srs._h, _ptr(seed), ctypes.byref(h)))
        self._h = h

    def add(self, vk, instance, instance_len, proofs, ctx=None):
        """add_proof for each of `proofs` (byte strings of one length, at most 4096) of vk's circuit; instance / instance_len
        as in VerifyingKey.verify_batch.  A proof that fails before its final check makes finalize() False.  With `proofs` a
        CUDA tensor (and `instance` one, as in VerifyingKey.verify_batch_dev) the add runs on the device
        (tb_dev_batch_verifier_add) and returns without waiting."""
        ctx = ctx or self.ctx
        if hasattr(proofs, "is_cuda") and proofs.is_cuda:
            B, inst, lens, addr, stride, plen = _dev_args(ctx, instance, instance_len, proofs, None)
            ctx._check(ctx._lib.tb_dev_batch_verifier_add(ctx._h, self._h, vk._h, B, inst, _ptr(lens), addr, stride, plen))
        else:
            B, inst, lens, buf, stride, plen = _host_args(instance, instance_len, proofs)
            ctx._check(ctx._lib.tb_batch_verifier_add(ctx._h, self._h, vk._h, B, _ptr(inst), _ptr(lens), _ptr(buf), stride, plen))

    def finalize(self, ctx=None):
        """True iff every proof added would be accepted by VerifyingKey.verify_batch.  Consumes the batch."""
        ctx = ctx or self.ctx
        ok = np.zeros(1, np.uint8)
        ctx._check(ctx._lib.tb_batch_verifier_finalize(ctx._h, self._h, _ptr(ok)))
        return bool(ok[0])

    def close(self):
        if getattr(self, "_h", None):
            self.ctx._lib.tb_batch_verifier_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
