//! Safe wrapper over `valida-b200-sys`.
//!
//! * [`Context`] — one per device: `StarkConfigImpl::new(pcs, challenger)` of the reference (`machine/src/config.rs:33-49`)
//!   becomes `Context::new(device)` + [`Context::set_challenger`] with the Poseidon round constants the caller drew
//!   (`basic/src/bin/valida.rs:360-365`).
//! * [`Context::prove_bytes`] — the body of `Machine::prove` (`derive/src/lib.rs:275-446`) from the 14 main and 2
//!   preprocessed traces to the CBOR image of `MachineProof` (`ciborium::into_writer`, `valida.rs:425-426`).
//! * [`Context::verify_bytes`] — `Machine::verify` (`derive/src/lib.rs:492-650`) on the same bytes.
//! * [`LocalGroup`] — ONE proof split across several GPUs, a worker thread per GPU inside this process.
//! * `--features valida`: [`glue::prove`] / [`glue::verify`] with the reference's own types.
//!
//! NOT COMPILED in the container this repository is developed in (no Rust toolchain there); the C caller
//! `tests/c/c_abi_smoke.c` exercises the same ABI and is built and run by the test suite.

use std::ffi::{c_void, CStr};
use std::fmt;
use std::marker::PhantomData;
use std::ptr;

pub use valida_b200_sys as sys;
use sys::{vgpu_ctx, vgpu_dev_matrix, vgpu_dmat, vgpu_matrix};

/// An error reported by the library (status code + `vgpu_last_error` text).  The reference's prover panics on failure
/// (`derive/src/lib.rs:319,364,396`); callers that want that behaviour `unwrap()`.
#[derive(Debug, Clone)]
pub struct Error {
    pub code: i32,
    pub message: String,
}

impl fmt::Display for Error {
    fn fmt(&self, f: &mut fmt::Formatter<'_>) -> fmt::Result {
        write!(f, "valida_b200 error {}: {}", self.code, self.message)
    }
}
impl std::error::Error for Error {}

pub type Result<T> = std::result::Result<T, Error>;

/// Word representation of the BabyBear elements that cross the boundary.
#[derive(Clone, Copy, Debug, PartialEq, Eq)]
pub enum Repr {
    /// `0 <= x < p`
    Canonical,
    /// `x * 2^32 mod p` — the `value` field of `p3_baby_bear::BabyBear`, so `RowMajorMatrix<BabyBear>.values` crosses zero-copy.
    MontyR32,
}

impl Repr {
    fn raw(self) -> i32 {
        match self {
            Repr::Canonical => sys::VGPU_REPR_CANONICAL,
            Repr::MontyR32 => sys::VGPU_REPR_MONTY_R32,
        }
    }
}

/// The hash of the Merkle trees (the `ValMmcs` of the `StarkConfig`), chosen with [`Context::set_merkle_hash`].
#[derive(Clone, Copy, Debug, PartialEq, Eq)]
pub enum MerkleHash {
    /// `FieldMerkleTreeMmcs<Val, SerializingHasher32<Keccak256Hash>, CompressionFunctionFromHasher<_, _, 2, 8>, 8>` (the default).
    Keccak256,
    /// `FieldMerkleTreeMmcs<Val, PaddingFreeSponge<Perm16, 16, 8, 8>, TruncatedPermutation<Perm16, 2, 8, 16>, 8>` over the
    /// challenger's Poseidon-16 instance.
    Poseidon16,
}

impl MerkleHash {
    fn raw(self) -> i32 {
        match self {
            MerkleHash::Keccak256 => sys::VGPU_MERKLE_KECCAK256,
            MerkleHash::Poseidon16 => sys::VGPU_MERKLE_POSEIDON16,
        }
    }
}

/// A borrowed row-major matrix of field words (`RowMajorMatrix<Val>`).
#[derive(Clone, Copy)]
pub struct MatrixView<'a> {
    pub values: &'a [u32],
    pub width: usize,
}

impl<'a> MatrixView<'a> {
    pub fn new(values: &'a [u32], width: usize) -> Self {
        assert!(width > 0 && values.len() % width == 0, "values.len() must be a multiple of the width");
        Self { values, width }
    }
    pub fn height(&self) -> usize {
        self.values.len() / self.width
    }
    fn raw(&self) -> vgpu_matrix {
        vgpu_matrix { data: self.values.as_ptr(), height: self.height() as u64, width: self.width as u64 }
    }
}

/// A strided matrix of field words in device memory of the context's device (a buffer the caller's own kernels filled).  Strides
/// count elements: element `(r, c)` is at `ptr[r * row_stride + c * col_stride]`.
#[derive(Clone, Copy, Debug)]
pub struct DeviceView {
    pub ptr: *const u32,
    pub height: u64,
    pub width: u64,
    pub row_stride: u64,
    pub col_stride: u64,
}

impl DeviceView {
    pub fn row_major(ptr: *const u32, height: u64, width: u64) -> Self {
        Self { ptr, height, width, row_stride: width, col_stride: 1 }
    }
    pub fn col_major(ptr: *const u32, height: u64, width: u64) -> Self {
        Self { ptr, height, width, row_stride: 1, col_stride: height }
    }
    fn raw(&self) -> vgpu_dev_matrix {
        vgpu_dev_matrix { data: self.ptr, height: self.height, width: self.width, row_stride: self.row_stride, col_stride: self.col_stride }
    }
}

/// A matrix on the device, in the library's layout: imported (a library-owned copy) or borrowed (the caller's buffer, read in
/// place).  It cannot outlive the [`Context`] it was made on; dropping it releases the handle (never a borrowed buffer).
pub struct DMat<'ctx> {
    raw: *mut vgpu_dmat,
    _ctx: PhantomData<&'ctx Context>,
}

impl DMat<'_> {
    pub fn as_ptr(&self) -> *const vgpu_dmat {
        self.raw
    }

    /// Logical (height, width).
    pub fn dims(&self) -> (u64, u64) {
        let (mut h, mut w) = (0u64, 0u64);
        unsafe { sys::vgpu_dmat_dims(self.raw, &mut h, &mut w) };
        (h, w)
    }

    /// Writes the rows held here into the caller's `height x width` view, in natural row order and `repr` words, on the context's
    /// stream without a host synchronisation; order a consumer after it with [`Context::record_event`].
    ///
    /// # Safety
    /// `dst` must describe writable device memory of `ctx`'s device that nothing else reads or writes until the export has run.
    pub unsafe fn export_device(&self, ctx: &Context, repr: Repr, dst: &DeviceView) -> Result<()> {
        let raw = dst.raw();
        ctx.check(sys::vgpu_dmat_export(ctx.raw, self.raw, repr.raw(), &raw))
    }

    /// The rows held on this rank (`row0`, `rows`): all of them unless the matrix is a row shard of a split proof.
    pub fn local_rows(&self) -> (u64, u64) {
        let (mut row0, mut rows) = (0u64, 0u64);
        unsafe { sys::vgpu_dmat_local_rows(self.raw, &mut row0, &mut rows) };
        (row0, rows)
    }

    /// Writes the rows held on this rank into the caller's `rows x width` view (local row `i` at row `i`), in `repr` words, on the
    /// context's stream without a host synchronisation; of a whole matrix the same as [`DMat::export_device`].
    ///
    /// # Safety
    /// As for [`DMat::export_device`].
    pub unsafe fn export_device_local(&self, ctx: &Context, repr: Repr, dst: &DeviceView) -> Result<()> {
        let raw = dst.raw();
        ctx.check(sys::vgpu_dmat_export_local(ctx.raw, self.raw, repr.raw(), &raw))
    }
}

impl Drop for DMat<'_> {
    fn drop(&mut self) {
        unsafe { sys::vgpu_dmat_free(self.raw) }
    }
}

/// Outcome of [`Context::verify_bytes`]: `Machine::verify` returns `Result<(), ()>`; the code says which check failed.
#[derive(Clone, Copy, Debug, PartialEq, Eq)]
pub enum Verdict {
    Accept,
    /// `VGPU_REJECT_*` of `include/valida_b200.h`; `-100 - chip` is the reference's `OodEvaluationMismatch` of that chip.
    Reject(i32),
}

/// One context per device and stream.  Not `Sync`: a context is single-threaded (a thread per GPU uses a context each).
pub struct Context {
    raw: *mut vgpu_ctx,
}

// A context may move to the worker thread that drives its GPU.
unsafe impl Send for Context {}

impl Context {
    /// `device`: CUDA ordinal.  The library owns its stream; fails when no CUDA device is present (there is no CPU fallback).
    pub fn new(device: i32) -> Result<Self> {
        let mut raw: *mut vgpu_ctx = ptr::null_mut();
        let code = unsafe { sys::vgpu_ctx_create(device, ptr::null_mut(), &mut raw) };
        if raw.is_null() {
            return Err(Error { code, message: "vgpu_ctx_create returned no context".into() });
        }
        let ctx = Context { raw };
        if code != 0 {
            return Err(ctx.error(code));      // dropping `ctx` destroys the half-made context
        }
        Ok(ctx)
    }

    pub fn as_ptr(&self) -> *mut vgpu_ctx {
        self.raw
    }

    fn error(&self, code: i32) -> Error {
        let message = unsafe {
            let p = sys::vgpu_last_error(self.raw);
            if p.is_null() { String::new() } else { CStr::from_ptr(p).to_string_lossy().into_owned() }
        };
        Error { code, message }
    }

    fn check(&self, code: i32) -> Result<()> {
        if code == 0 { Ok(()) } else { Err(self.error(code)) }
    }

    /// The Poseidon instance of the `DuplexChallenger`: 480 round constants (canonical words, `perm16.constants()` order) and
    /// the 16 x 16 MDS matrix row-major, or `None` for `CosetMds<_, 16>::default()`.
    pub fn set_challenger(&mut self, round_constants: &[u32; 480], mds: Option<&[u32; 256]>) -> Result<()> {
        let mds_ptr = mds.map_or(ptr::null(), |m| m.as_ptr());
        self.check(unsafe { sys::vgpu_set_challenger(self.raw, round_constants.as_ptr(), mds_ptr) })
    }

    /// The Merkle tree hash of the commits, openings, proofs and verifications that follow.  `Poseidon16` uses the instance of
    /// [`Context::set_challenger`], which must come first.  Proof bytes keep their format; a proof verifies only under the hash
    /// it was made with.
    pub fn set_merkle_hash(&mut self, hash: MerkleHash) -> Result<()> {
        self.check(unsafe { sys::vgpu_ctx_set_merkle_hash(self.raw, hash.raw()) })
    }

    /// Debug mode of [`Context::prove_bytes`] (off by default): every chip's constraints on every trace row and the cumulative sums
    /// are checked before the commitments, as the reference's `prove` does in debug builds; a bad witness is an error naming each
    /// failing chip, row and constraint.  `Machine::prove` passes `cfg!(debug_assertions)`.
    pub fn set_debug_checks(&mut self, on: bool) -> Result<()> {
        self.check(unsafe { sys::vgpu_ctx_set_debug_checks(self.raw, on as i32) })
    }

    /// Page-locks a caller buffer in place so that the uploads of [`Context::prove_bytes`] overlap its commits.
    pub fn host_register(&mut self, words: &[u32]) -> Result<()> {
        self.check(unsafe { sys::vgpu_host_register(self.raw, words.as_ptr() as *const c_void, (words.len() * 4) as u64) })
    }
    pub fn host_unregister(&mut self, words: &[u32]) -> Result<()> {
        self.check(unsafe { sys::vgpu_host_unregister(self.raw, words.as_ptr() as *const c_void) })
    }

    /// `Machine::prove`: `main` are the 14 chip traces in BasicMachine order (`basic/src/lib.rs:151-166`), `prep` the
    /// preprocessed traces (program: 7 columns, range: 1 column).  Returns the CBOR image of `MachineProof`.
    pub fn prove_bytes(&mut self, main: &[MatrixView<'_>; sys::VGPU_NUM_CHIPS], prep: &[MatrixView<'_>; 2], repr: Repr) -> Result<Vec<u8>> {
        let main_raw: Vec<vgpu_matrix> = main.iter().map(MatrixView::raw).collect();
        let prep_raw: Vec<vgpu_matrix> = prep.iter().map(MatrixView::raw).collect();
        let (mut bytes, mut len) = (ptr::null_mut::<u8>(), 0u64);
        let code = unsafe { sys::vgpu_prove(self.raw, main_raw.as_ptr(), prep_raw.as_ptr(), repr.raw(), &mut bytes, &mut len) };
        self.check(code)?;
        let proof = unsafe { std::slice::from_raw_parts(bytes, len as usize) }.to_vec();
        unsafe { sys::vgpu_free_bytes(bytes) };
        Ok(proof)
    }

    /// `Machine::verify` on CBOR proof bytes (this library's or the reference's).
    pub fn verify_bytes(&mut self, proof: &[u8], prep: &[MatrixView<'_>; 2], repr: Repr) -> Result<Verdict> {
        let prep_raw: Vec<vgpu_matrix> = prep.iter().map(MatrixView::raw).collect();
        let mut verdict = -1i32;
        let code = unsafe { sys::vgpu_verify(self.raw, proof.as_ptr(), proof.len() as u64, prep_raw.as_ptr(), repr.raw(), &mut verdict) };
        self.check(code)?;
        Ok(if verdict == sys::VGPU_ACCEPT { Verdict::Accept } else { Verdict::Reject(verdict) })
    }

    /// Copies a device matrix the caller holds (any strides, `repr` words) into a library-owned one, on the context's stream.
    /// Every word must be below p: otherwise the error names the first offending (row, column) and nothing is created.
    /// Synchronises the context's stream once; the caller's buffer may change as soon as this returns.
    ///
    /// # Safety
    /// `src` must describe readable device memory of this context's device, and whatever writes it must be ordered before the
    /// context's stream (the same stream, or [`Context::wait_event`]).
    pub unsafe fn import_device(&self, src: &DeviceView, repr: Repr) -> Result<DMat<'_>> {
        let raw = src.raw();
        let mut out: *mut vgpu_dmat = ptr::null_mut();
        self.check(sys::vgpu_dmat_import(self.raw, &raw, repr.raw(), &mut out))?;
        Ok(DMat { raw: out, _ctx: PhantomData })
    }

    /// [`Context::import_device`] for a rank of a [`LocalGroup`]: every rank passes a view of the whole matrix on its own device,
    /// and of a trace tall enough to be split only this rank's run of rows is read.
    ///
    /// # Safety
    /// As for [`Context::import_device`].
    pub unsafe fn import_device_rows(&self, src: &DeviceView, repr: Repr) -> Result<DMat<'_>> {
        let raw = src.raw();
        let mut out: *mut vgpu_dmat = ptr::null_mut();
        self.check(sys::vgpu_dmat_import_rows(self.raw, &raw, repr.raw(), &mut out))?;
        Ok(DMat { raw: out, _ctx: PhantomData })
    }

    /// Zero-copy: the caller's column-major Montgomery buffer (element `(r, c)` at `data[c * col_stride + r]`, `col_stride >=
    /// height`, 4-byte aligned) is proven from in place.  One read pass checks every word is below p; nothing is copied.
    ///
    /// # Safety
    /// The library never writes or frees `data`, but reads it whenever a call takes the returned [`DMat`].  The caller keeps the
    /// buffer allocated and unchanged until the `DMat` is dropped AND every call that took it has returned; writes to it before the
    /// borrow must be ordered before the context's stream.
    pub unsafe fn borrow_device(&self, data: *mut u32, height: u64, width: u64, col_stride: u64) -> Result<DMat<'_>> {
        let mut out: *mut vgpu_dmat = ptr::null_mut();
        self.check(sys::vgpu_dmat_borrow(self.raw, data, height, width, col_stride, &mut out))?;
        Ok(DMat { raw: out, _ctx: PhantomData })
    }

    /// The rows `(row0, rows)` this rank holds of a matrix of logical height `height`, and so must supply to
    /// [`Context::import_device_local`] and [`Context::borrow_device_local`]: its run of a trace tall enough to be split, otherwise
    /// `(0, height)`.  Known before any matrix exists, so each rank can fill only its own rows.
    pub fn local_rows(&self, height: u64) -> (u64, u64) {
        let (mut row0, mut rows) = (0u64, 0u64);
        unsafe { sys::vgpu_ctx_local_rows(self.raw, height, &mut row0, &mut rows) };
        (row0, rows)
    }

    /// [`Context::import_device`] of this rank's rows only: `local` views the `rows` of [`Context::local_rows`]`(height)` (any
    /// strides), local row `i` being row `row0 + i` of the matrix.  The result equals [`Context::import_device_rows`] of a view of
    /// the whole matrix; a word not below p fails on this rank only, naming its row in the whole matrix.
    ///
    /// # Safety
    /// As for [`Context::import_device`].
    pub unsafe fn import_device_local(&self, local: &DeviceView, height: u64, repr: Repr) -> Result<DMat<'_>> {
        let raw = local.raw();
        let mut out: *mut vgpu_dmat = ptr::null_mut();
        self.check(sys::vgpu_dmat_import_local(self.raw, &raw, height, repr.raw(), &mut out))?;
        Ok(DMat { raw: out, _ctx: PhantomData })
    }

    /// [`Context::borrow_device`] of this rank's rows only: `data` holds the `rows` of [`Context::local_rows`]`(height)`, column-major
    /// Montgomery (local row `i` of column `c` at `data[c * col_stride + i]`, `col_stride >= rows`, 4-byte aligned), and is proven
    /// from in place.
    ///
    /// # Safety
    /// As for [`Context::borrow_device`]: the library never writes or frees `data`; the caller keeps it allocated and unchanged until
    /// the `DMat` is dropped AND every call that took it has returned, and orders writes to it before the context's stream.
    pub unsafe fn borrow_device_local(&self, data: *mut u32, height: u64, width: u64, col_stride: u64) -> Result<DMat<'_>> {
        let mut out: *mut vgpu_dmat = ptr::null_mut();
        self.check(sys::vgpu_dmat_borrow_local(self.raw, data, height, width, col_stride, &mut out))?;
        Ok(DMat { raw: out, _ctx: PhantomData })
    }

    /// The context's stream waits for `cuda_event` (a `cudaEvent_t` the caller recorded on a producer stream).
    ///
    /// # Safety
    /// `cuda_event` must be a valid CUDA event of this context's device.
    pub unsafe fn wait_event(&self, cuda_event: *mut c_void) -> Result<()> {
        self.check(sys::vgpu_ctx_wait_event(self.raw, cuda_event))
    }

    /// Records `cuda_event` on the context's stream, for a consumer stream to wait for (after [`DMat::export_device`]).
    ///
    /// # Safety
    /// As for [`Context::wait_event`].
    pub unsafe fn record_event(&self, cuda_event: *mut c_void) -> Result<()> {
        self.check(sys::vgpu_ctx_record_event(self.raw, cuda_event))
    }

    /// The handle arrays of a machine witness (14 main and 2 preprocessed traces), as the calls that take one want them.
    fn witness_ptrs(main: &[&DMat<'_>; sys::VGPU_NUM_CHIPS], prep: &[&DMat<'_>; 2]) -> ([*const vgpu_dmat; sys::VGPU_NUM_CHIPS], [*const vgpu_dmat; 2]) {
        (std::array::from_fn(|i| main[i].as_ptr()), std::array::from_fn(|i| prep[i].as_ptr()))
    }

    /// `Machine::prove` from traces already on the device (imported or borrowed): the same bytes as [`Context::prove_bytes`].
    pub fn prove_device_bytes(&self, main: &[&DMat<'_>; sys::VGPU_NUM_CHIPS], prep: &[&DMat<'_>; 2]) -> Result<Vec<u8>> {
        let (main_raw, prep_raw) = Self::witness_ptrs(main, prep);
        let (mut bytes, mut len) = (ptr::null_mut::<u8>(), 0u64);
        let code = unsafe { sys::vgpu_prove_device(self.raw, main_raw.as_ptr(), prep_raw.as_ptr(), &mut bytes, &mut len) };
        self.check(code)?;
        let proof = unsafe { std::slice::from_raw_parts(bytes, len as usize) }.to_vec();
        unsafe { sys::vgpu_free_bytes(bytes) };
        Ok(proof)
    }

    /// `check_constraints` (`machine/src/check_constraints.rs:14-84`) of BasicMachine chip `chip_id` on a rank of a split proof:
    /// every rank passes its own matrices (its row shards of the tall traces, or whole matrices) and gets what the check of the
    /// whole traces on one GPU gives: `(first failing row or -1, its first failing constraint, number of failing rows)`.  On a
    /// context that does not split proofs it is the single-GPU check.  Collective; synchronises.
    pub fn check_constraints_local(&self, chip_id: u32, main: &DMat<'_>, prep: Option<&DMat<'_>>, perm: &DMat<'_>, challenges: &[u32; 15]) -> Result<(i64, u32, u64)> {
        let chip = unsafe { sys::vgpu_basic_machine_chip(chip_id) };
        let prep_ptr = prep.map_or(ptr::null(), |m| m.as_ptr());
        let (mut row, mut constraint, mut failing) = (0i64, 0u32, 0u64);
        self.check(unsafe {
            sys::vgpu_check_constraints_local(self.raw, chip, main.as_ptr(), prep_ptr, perm.as_ptr(), challenges.as_ptr(), &mut row, &mut constraint, &mut failing)
        })?;
        Ok((row, constraint, failing))
    }

    /// Every `(row, constraint, value)` on which the check of [`Context::check_constraints_local`] does not vanish, not only the first:
    /// the first `min(cap, total)` in ascending (row, constraint) order, the total, and per constraint (eval order) the number of rows
    /// on which it fails.  Same arguments and refusals as `check_constraints_local`; collective on a split context, with the same
    /// result on every rank.  Synchronises.
    pub fn check_failures(&self, chip_id: u32, main: &DMat<'_>, prep: Option<&DMat<'_>>, perm: &DMat<'_>, challenges: &[u32; 15], cap: usize)
                          -> Result<(Vec<sys::vgpu_check_failure>, u64, Vec<u64>)> {
        let chip = unsafe { sys::vgpu_basic_machine_chip(chip_id) };
        let (mut air, mut total_constraints) = (0u32, 0u32);
        if unsafe { sys::vgpu_chip_constraint_count(chip, &mut air, &mut total_constraints) } != 0 {
            return Err(Error { code: -1, message: format!("check_failures: unknown chip id {chip_id}") });
        }
        let prep_ptr = prep.map_or(ptr::null(), |m| m.as_ptr());
        let mut out = vec![sys::vgpu_check_failure::default(); cap];
        let mut per = vec![0u64; total_constraints as usize];
        let (mut n, mut total) = (0u64, 0u64);
        self.check(unsafe {
            sys::vgpu_check_failures(self.raw, chip, main.as_ptr(), prep_ptr, perm.as_ptr(), challenges.as_ptr(), cap as u64, out.as_mut_ptr(),
                                     &mut n, &mut total, per.as_mut_ptr())
        })?;
        out.truncate(n as usize);
        Ok((out, total, per))
    }

    /// Every main-trace cell of one chip's witness that no check pins (no `Air::eval` assertion and no bus event changes with it):
    /// the first `min(cap, total)` in ascending (row, column) order, the total, and per column the number of free rows.  Takes what
    /// [`Context::check_failures`] takes without the permutation trace and the challenges, and refuses the same traces; collective
    /// on a split context, with the same result on every rank.  Synchronises.
    pub fn free_cells(&self, chip_id: u32, main: &DMat<'_>, prep: Option<&DMat<'_>>, cap: usize) -> Result<(Vec<sys::vgpu_free_cell>, u64, Vec<u64>)> {
        let chip = unsafe { sys::vgpu_basic_machine_chip(chip_id) };
        if chip.is_null() {
            return Err(Error { code: -1, message: format!("free_cells: unknown chip id {chip_id}") });
        }
        let width = unsafe { (*chip).width } as usize;
        let prep_ptr = prep.map_or(ptr::null(), |m| m.as_ptr());
        let mut out = vec![sys::vgpu_free_cell::default(); cap];
        let mut per = vec![0u64; width];
        let (mut n, mut total) = (0u64, 0u64);
        self.check(unsafe {
            sys::vgpu_free_cells(self.raw, chip, main.as_ptr(), prep_ptr, cap as u64, out.as_mut_ptr(), &mut n, &mut total, per.as_mut_ptr())
        })?;
        out.truncate(n as usize);
        Ok((out, total, per))
    }

    /// Every main-trace cell of one chip's witness that the chip's `Air::eval` assertions would also accept at another value (the
    /// assertions that depend on the cell share a root other than its value), with those values: the first `min(cap, total)` in
    /// ascending (row, column) order, the total, the number whose `bus` is 0, and per column the listed rows followed by the bus-free
    /// ones (`2 * width` entries).  Takes what [`Context::free_cells`] takes and refuses the same traces; collective on a split
    /// context, with the same result on every rank.  Synchronises.
    pub fn cell_alternatives(&self, chip_id: u32, main: &DMat<'_>, prep: Option<&DMat<'_>>, cap: usize) -> Result<(Vec<sys::vgpu_cell_alternative>, u64, u64, Vec<u64>)> {
        let chip = unsafe { sys::vgpu_basic_machine_chip(chip_id) };
        if chip.is_null() {
            return Err(Error { code: -1, message: format!("cell_alternatives: unknown chip id {chip_id}") });
        }
        let width = unsafe { (*chip).width } as usize;
        let prep_ptr = prep.map_or(ptr::null(), |m| m.as_ptr());
        let mut out = vec![sys::vgpu_cell_alternative::default(); cap];
        let mut per = vec![0u64; 2 * width];
        let (mut n, mut total, mut bus_free) = (0u64, 0u64, 0u64);
        self.check(unsafe {
            sys::vgpu_cell_alternatives(self.raw, chip, main.as_ptr(), prep_ptr, cap as u64, out.as_mut_ptr(), &mut n, &mut total, &mut bus_free, per.as_mut_ptr())
        })?;
        out.truncate(n as usize);
        Ok((out, total, bus_free, per))
    }

    /// The witness check of the reference's debug builds (`check_constraints` of every chip + `check_cumulative_sums`,
    /// `derive/src/lib.rs:246-253,376-377`) without a proof, with the caller's 15 challenge words: one report per chip and whether
    /// the cumulative sums cancel.  `main` / `prep` are whole traces or, on a [`LocalGroup`] rank, its row shards; every rank of a
    /// split proof makes the call and gets the same reports.  A host that splits proofs runs this in debug builds.
    pub fn check_witness(&self, main: &[&DMat<'_>; sys::VGPU_NUM_CHIPS], prep: &[&DMat<'_>; 2], challenges: &[u32; 15]) -> Result<([sys::vgpu_check_report; sys::VGPU_NUM_CHIPS], bool)> {
        let (main_raw, prep_raw) = Self::witness_ptrs(main, prep);
        let mut reports = [sys::vgpu_check_report::default(); sys::VGPU_NUM_CHIPS];
        let mut cancel = 0i32;
        self.check(unsafe { sys::vgpu_check_witness(self.raw, main_raw.as_ptr(), prep_raw.as_ptr(), challenges.as_ptr(), reports.as_mut_ptr(), &mut cancel) })?;
        Ok((reports, cancel != 0))
    }

    /// Every bus tuple the witness leaves unbalanced, with every event that sends or receives it: the tuples in ascending (bus,
    /// fields) order, the events (tuple `t`'s at `t.first_event..t.first_event + t.n_events`, ascending by (chip, row, interaction))
    /// and the number of candidate groups whose events did not fit under `cap` (0: the list is complete).  Takes what
    /// [`Context::check_witness`] takes; collective on a split context, with the same result on every rank.  Synchronises.
    pub fn check_buses(&self, main: &[&DMat<'_>; sys::VGPU_NUM_CHIPS], prep: &[&DMat<'_>; 2], challenges: &[u32; 15], cap: usize)
                       -> Result<(Vec<sys::vgpu_bus_imbalance>, Vec<sys::vgpu_bus_event>, u64)> {
        let (main_raw, prep_raw) = Self::witness_ptrs(main, prep);
        let mut tuples = vec![sys::vgpu_bus_imbalance::default(); cap];
        let mut events = vec![sys::vgpu_bus_event::default(); cap];
        let (mut nt, mut ne, mut unexamined) = (0u64, 0u64, 0u64);
        self.check(unsafe {
            sys::vgpu_check_buses(self.raw, main_raw.as_ptr(), prep_raw.as_ptr(), challenges.as_ptr(), cap as u64, tuples.as_mut_ptr(), &mut nt,
                                  events.as_mut_ptr(), &mut ne, &mut unexamined)
        })?;
        tuples.truncate(nt as usize);
        events.truncate(ne as usize);
        Ok((tuples, events, unexamined))
    }

    /// Every event of the witness that carries each item's bus tuple, sends and receives alike (the items' `multiplicity` and
    /// `is_send` are ignored, so the events of [`Context::check_buses`] and of this call are items as they are): one link per item
    /// (its tuple, its own count, the summed send and receive multiplicities and the number of events carrying the tuple, exact), the
    /// events of the listed tuples (tuple order ascending by (bus, fields), each tuple's events ascending by (chip, row, interaction),
    /// shared by the items with that tuple; an unlisted tuple's `first_event` is `u64::MAX`) and the number of distinct tuples whose
    /// events did not fit under `cap`.  Takes what [`Context::check_buses`] takes; collective on a split context, with the same result
    /// on every rank.  Synchronises.
    pub fn bus_links(&self, main: &[&DMat<'_>; sys::VGPU_NUM_CHIPS], prep: &[&DMat<'_>; 2], items: &[sys::vgpu_bus_event], cap: usize)
                     -> Result<(Vec<sys::vgpu_bus_link>, Vec<sys::vgpu_bus_event>, u64)> {
        let (main_raw, prep_raw) = Self::witness_ptrs(main, prep);
        let mut links = vec![sys::vgpu_bus_link::default(); items.len()];
        let mut events = vec![sys::vgpu_bus_event::default(); cap];
        let (mut ne, mut unlisted) = (0u64, 0u64);
        self.check(unsafe {
            sys::vgpu_bus_links(self.raw, main_raw.as_ptr(), prep_raw.as_ptr(), items.as_ptr(), items.len() as u64, links.as_mut_ptr(), cap as u64,
                                events.as_mut_ptr(), &mut ne, &mut unlisted)
        })?;
        events.truncate(ne as usize);
        Ok((links, events, unlisted))
    }

    /// The values of the cells each `(row, constraint)` item reads (the items' `value` fields are ignored: [`Context::check_failures`]'
    /// list as it is; a bus event of [`Context::check_buses`] is `(row, air_constraints + interaction)`), per item in
    /// [`constraint_cells`] order, canonical; a next-row cell is read at `(row + 1) mod h`.  Without `perm` the permutation cells are
    /// `None`.  Takes what `check_failures` takes and refuses the same traces, a row or constraint out of range, before anything is
    /// enqueued; collective on a split context (every rank passes the same items and gets the same values).  Synchronises once.
    pub fn explain_failures(&self, chip_id: u32, main: &DMat<'_>, prep: Option<&DMat<'_>>, perm: Option<&DMat<'_>>,
                            items: &[sys::vgpu_check_failure]) -> Result<Vec<Vec<Option<u32>>>> {
        let chip = unsafe { sys::vgpu_basic_machine_chip(chip_id) };
        let mut need = 0u64;
        for it in items {
            // an item out of range is left for the call to refuse, naming it
            need += constraint_cells(chip_id, it.constraint).map_or(0, |(_, c)| c.len() as u64);
        }
        let mut first = vec![0u64; items.len() + 1];
        let mut values = vec![0u32; need.max(1) as usize];
        let mut n_values = 0u64;
        self.check(unsafe {
            sys::vgpu_explain_failures(self.raw, chip, main.as_ptr(), prep.map_or(ptr::null(), |m| m.as_ptr()), perm.map_or(ptr::null(), |m| m.as_ptr()),
                                       items.as_ptr(), items.len() as u64, first.as_mut_ptr(), values.as_mut_ptr(), need, &mut n_values)
        })?;
        Ok((0..items.len())
            .map(|i| values[first[i] as usize..first[i + 1] as usize].iter().map(|&v| if v == sys::VGPU_CELL_ABSENT { None } else { Some(v) }).collect())
            .collect())
    }

    /// Every cell of the witness `main` / `prep` that differs from what `Chip::generate_trace` writes for the run `log` records:
    /// the first `min(cap, total)` cells in ascending (chip, trace, row, column) order (so the first CPU cell is on the first cycle
    /// whose row differs), their total, one summary per chip (a chip whose height differs from the run's is reported there and not
    /// compared) and the differing cells of each column ([`witness_column_count`] entries).  Takes what [`Context::check_buses`]
    /// takes; collective on a split context, with the same result on every rank.  The expected witness is built and compared on the
    /// device one chip at a time.  Synchronises.
    pub fn diff_witness(&self, log: &VmLog, main: &[&DMat<'_>; sys::VGPU_NUM_CHIPS], prep: &[&DMat<'_>; 2], cap: usize)
                        -> Result<(Vec<sys::vgpu_cell_diff>, u64, [sys::vgpu_diff_summary; sys::VGPU_NUM_CHIPS], Vec<u64>)> {
        let (main_raw, prep_raw) = Self::witness_ptrs(main, prep);
        let mut out = vec![sys::vgpu_cell_diff::default(); cap];
        let mut summary = [sys::vgpu_diff_summary::default(); sys::VGPU_NUM_CHIPS];
        let mut per_column = vec![0u64; witness_column_count()];
        let (mut n, mut total) = (0u64, 0u64);
        self.check(unsafe {
            sys::vgpu_diff_witness(self.raw, log.raw, main_raw.as_ptr(), prep_raw.as_ptr(), cap as u64, out.as_mut_ptr(), &mut n, &mut total,
                                   summary.as_mut_ptr(), per_column.as_mut_ptr())
        })?;
        out.truncate(n as usize);
        Ok((out, total, summary, per_column))
    }

    /// Kernels launched by this context so far.
    pub fn launch_count(&self) -> u64 {
        unsafe { sys::vgpu_ctx_launch_count(self.raw) }
    }

    /// Device memory of this context in bytes; `reset` restarts both peaks from the current live bytes.
    pub fn memory_stats(&mut self, reset: bool) -> Result<MemoryStats> {
        let mut out = [0u64; 4];
        self.check(unsafe { sys::vgpu_ctx_memory_stats(self.raw, out.as_mut_ptr(), reset as i32) })?;
        Ok(MemoryStats { live: out[0], peak: out[1], cached: out[2], symm_peak: out[3] })
    }
}

/// The name of a column of a BasicMachine chip's trace (`sys::VGPU_TRACE_MAIN`, `VGPU_TRACE_PREPROCESSED` or `VGPU_TRACE_PERMUTATION`),
/// after the reference's column structs (e.g. `mem_channels[1].value[2]`); `None` out of range.  Host only.
pub fn column_name(chip_id: u32, trace: u32, column: u32) -> Option<String> {
    let p = unsafe { sys::vgpu_chip_column_name(sys::vgpu_basic_machine_chip(chip_id), trace as i32, column) };
    if p.is_null() { None } else { Some(unsafe { CStr::from_ptr(p) }.to_string_lossy().into_owned()) }
}

/// Constraint `constraint` of a BasicMachine chip (eval order, as [`Context::check_failures`] numbers it): its label (the block of the
/// reference's eval for an AIR assertion, e.g. `CpuChip::eval_pc`) and the cells it reads, in ascending (trace, next, column) order.
/// Host only.
pub fn constraint_cells(chip_id: u32, constraint: u32) -> Result<(String, Vec<sys::vgpu_cell>)> {
    let chip = unsafe { sys::vgpu_basic_machine_chip(chip_id) };
    let mut label: *const std::ffi::c_char = ptr::null();
    let mut n = 0u32;
    let refused = || Error { code: -1, message: format!("constraint_cells: chip {chip_id} has no constraint {constraint}") };
    if unsafe { sys::vgpu_chip_constraint_cells(chip, constraint, &mut label, ptr::null_mut(), 0, &mut n) } != 0 {
        return Err(refused());
    }
    let mut cells = vec![sys::vgpu_cell::default(); n as usize];
    if unsafe { sys::vgpu_chip_constraint_cells(chip, constraint, &mut label, cells.as_mut_ptr(), n, &mut n) } != 0 {
        return Err(refused());
    }
    Ok((unsafe { CStr::from_ptr(label) }.to_string_lossy().into_owned(), cells))
}

/// The length of [`Context::diff_witness`]' per-column counts: the main columns of chips 0..13 in chip order, then the 7 program and
/// the 1 range preprocessed columns.  Host only.
pub fn witness_column_count() -> usize {
    unsafe { sys::vgpu_witness_column_count() as usize }
}

/// The logs of one run of `Machine::run` (the interpreter on the host): what the device witness builder and
/// [`Context::diff_witness`] expand into the traces.
pub struct VmLog {
    raw: *mut sys::vgpu_vmlog,
}

unsafe impl Send for VmLog {}
unsafe impl Sync for VmLog {}

impl VmLog {
    /// Runs `program` (`n_instr` x 6 words: opcode, a, b, c, d, e) with the static cells `(address, value)` preloaded, ascending by address.
    pub fn run(program: &[[i32; 6]], initial_pc: u32, initial_fp: u32, max_cycles: u64, static_data: &[(u32, u32)]) -> Result<Self> {
        let addrs: Vec<u32> = static_data.iter().map(|&(a, _)| a).collect();
        let values: Vec<u32> = static_data.iter().map(|&(_, v)| v).collect();
        let mut raw = ptr::null_mut();
        let mut err = [0 as std::ffi::c_char; 512];
        let code = unsafe {
            sys::vgpu_vm_run(program.as_ptr() as *const i32, program.len() as u64, initial_pc, initial_fp, max_cycles, addrs.as_ptr(), values.as_ptr(),
                             static_data.len() as u64, &mut raw, err.as_mut_ptr(), err.len() as u64)
        };
        if code != 0 {
            return Err(Error { code, message: unsafe { CStr::from_ptr(err.as_ptr()) }.to_string_lossy().into_owned() });
        }
        Ok(VmLog { raw })
    }
}

impl Drop for VmLog {
    fn drop(&mut self) {
        unsafe { sys::vgpu_vmlog_free(self.raw) }
    }
}

/// What [`Context::memory_stats`] returns.
#[derive(Clone, Copy, Debug, PartialEq, Eq)]
pub struct MemoryStats {
    /// Buffers in use.
    pub live: u64,
    /// Peak of `live` since the context was created or the last reset.
    pub peak: u64,
    /// Freed buffers kept for reuse by later calls (emptied by `vgpu_ctx_release_cached`).
    pub cached: u64,
    /// Peak live bytes of the symmetric heap of a split proof (0 without one).
    pub symm_peak: u64,
}

impl Drop for Context {
    fn drop(&mut self) {
        unsafe { sys::vgpu_ctx_destroy(self.raw) }
    }
}

/// ONE proof split across the GPUs of a box: a context per device, a worker thread per context.  Every rank makes the same
/// call with the same traces and copies only its rows of the tall ones; the proof bytes are identical on all ranks and
/// identical to the single-GPU proof.  The number of ranks is 1..=16; at a count that is not a power
/// of two the ranks' row runs differ by at most one of 8 P units (P: the next power of two).
pub struct LocalGroup {
    ranks: Vec<Context>,
}

impl LocalGroup {
    /// `contexts[i]` becomes rank `i`; `set_challenger` must already have been called on each.
    pub fn new(contexts: Vec<Context>) -> Result<Self> {
        assert!(!contexts.is_empty());
        let raws: Vec<*mut vgpu_ctx> = contexts.iter().map(Context::as_ptr).collect();
        let code = unsafe { sys::vgpu_comm_init_local(raws.as_ptr(), raws.len() as i32) };
        contexts[0].check(code)?;
        Ok(LocalGroup { ranks: contexts })
    }

    pub fn len(&self) -> usize {
        self.ranks.len()
    }
    pub fn is_empty(&self) -> bool {
        self.ranks.is_empty()
    }

    /// One proof on all ranks; returns rank 0's bytes after checking that every rank produced the same ones.
    pub fn prove_bytes(&mut self, main: &[MatrixView<'_>; sys::VGPU_NUM_CHIPS], prep: &[MatrixView<'_>; 2], repr: Repr) -> Result<Vec<u8>> {
        let proofs: Vec<Result<Vec<u8>>> = std::thread::scope(|s| {
            let handles: Vec<_> = self.ranks.iter_mut().map(|ctx| s.spawn(move || ctx.prove_bytes(main, prep, repr))).collect();
            handles.into_iter().map(|h| h.join().expect("a rank's worker thread panicked")).collect()
        });
        let mut out: Option<Vec<u8>> = None;
        for p in proofs {
            let p = p?;
            match &out {
                None => out = Some(p),
                Some(first) => assert!(*first == p, "ranks disagree on the proof bytes"),
            }
        }
        Ok(out.unwrap())
    }
}

/// The reference's own types on top of the byte-level calls (`--features valida`).
#[cfg(feature = "valida")]
pub mod glue {
    use super::*;
    use p3_baby_bear::BabyBear;
    use p3_matrix::dense::RowMajorMatrix;
    use p3_matrix::Matrix;
    use valida_machine::{MachineProof, StarkConfig};

    /// `BabyBear` is `#[repr(transparent)]` over its Montgomery `u32` in the pinned fork, so the values slice is viewed in place.
    fn view(m: &RowMajorMatrix<BabyBear>) -> MatrixView<'_> {
        let words = unsafe { std::slice::from_raw_parts(m.values.as_ptr() as *const u32, m.values.len()) };
        MatrixView::new(words, m.width())
    }

    /// Replacement for the body of `Machine::prove` after witness generation (`derive/src/lib.rs:321-446`): the caller keeps
    /// steps 1-7 (`chips.par_iter().map(|c| c.generate_trace(self))`, `preprocessed_trace()`) and hands the traces over.
    pub fn prove<SC>(ctx: &mut Context, main_traces: &[RowMajorMatrix<BabyBear>; 14], preprocessed_traces: &[RowMajorMatrix<BabyBear>; 2]) -> MachineProof<SC>
    where
        SC: StarkConfig<Val = BabyBear>,
        MachineProof<SC>: serde::de::DeserializeOwned,
    {
        let main: Vec<MatrixView<'_>> = main_traces.iter().map(view).collect();
        let prep: Vec<MatrixView<'_>> = preprocessed_traces.iter().map(view).collect();
        let main: [MatrixView<'_>; 14] = main.try_into().ok().unwrap();
        let prep: [MatrixView<'_>; 2] = prep.try_into().ok().unwrap();
        let bytes = ctx.prove_bytes(&main, &prep, Repr::MontyR32).expect("vgpu_prove");   // the reference panics on failure too
        ciborium::from_reader(bytes.as_slice()).expect("proof decoding")
    }

    /// `Machine::verify` (`machine/src/machine.rs:26-31`): `Result<(), ()>` like the reference.
    pub fn verify<SC>(ctx: &mut Context, proof: &MachineProof<SC>, preprocessed_traces: &[RowMajorMatrix<BabyBear>; 2]) -> core::result::Result<(), ()>
    where
        SC: StarkConfig<Val = BabyBear>,
        MachineProof<SC>: serde::Serialize,
    {
        let mut bytes = Vec::new();
        ciborium::into_writer(proof, &mut bytes).map_err(|_| ())?;
        let prep: Vec<MatrixView<'_>> = preprocessed_traces.iter().map(view).collect();
        let prep: [MatrixView<'_>; 2] = prep.try_into().ok().unwrap();
        match ctx.verify_bytes(&bytes, &prep, Repr::MontyR32) {
            Ok(Verdict::Accept) => Ok(()),
            _ => Err(()),
        }
    }
}
