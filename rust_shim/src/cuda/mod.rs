//! `src/cuda/mod.rs` -- the file a RustFFT maintainer adds next to `src/avx/mod.rs`, `src/sse/mod.rs`.
//!
//! NOT COMPILED IN THIS REPOSITORY: the build image has no rustc/cargo.  It is the reference-side
//! binding for `include/b200fft.h`, written against RustFFT 6.4.1's backend plug-in pattern
//! (`src/sse/mod.rs:22-31`, `src/sse/sse_planner.rs:144-226`), and is what INTEGRATION.md walks through.

use std::any::TypeId;
use std::ffi::CStr;
use std::os::raw::{c_char, c_int, c_void};

use num_complex::Complex;

use crate::common::FftNum;
use crate::{Direction, Fft, FftDirection, Length};

pub mod cuda_dct;
pub mod cuda_planner;

#[repr(C)]
pub struct B200FftPlan {
    _private: [u8; 0],
}

#[link(name = "b200fft")]
extern "C" {
    pub fn b200fft_device_count(n: *mut c_int) -> c_int;
    pub fn b200fft_plan_create(out: *mut *mut B200FftPlan, len: u64, direction: c_int, precision: c_int, device: c_int) -> c_int;
    pub fn b200fft_plan_create_from_recipe(out: *mut *mut B200FftPlan, nodes: *const B200FftRecipeNode, n_nodes: u32, direction: c_int,
                                           precision: c_int, device: c_int) -> c_int;
    pub fn b200fft_plan_destroy(plan: *mut B200FftPlan) -> c_int;
    pub fn b200fft_exec_host_inplace(plan: *const B200FftPlan, buffer: *mut c_void, n_complex: u64) -> c_int;
    pub fn b200fft_exec_host_outofplace(plan: *const B200FftPlan, input: *const c_void, output: *mut c_void, n_complex: u64) -> c_int;
    pub fn b200fft_last_error() -> *const c_char;
}

/// `b200fft_recipe_node` of include/b200fft.h: the decomposition the Rust planner chose (`crate::plan::Recipe`,
/// src/plan.rs:134-226), flattened -- node 0 is the root, `child` is the inner FFT of a Rader / Bluestein node.
#[repr(C)]
#[derive(Clone, Copy)]
pub struct B200FftRecipeNode {
    pub kind: u32, // 0 auto, 1 pow2, 2 smooth, 3 mixed radix, 4 good-thomas, 5 rader, 6 bluestein
    pub child: u32,
    pub len: u64,
    pub a: u64,
    pub b: u64,
}

pub(crate) fn last_error_text() -> String {
    last_error()
}

fn last_error() -> String {
    unsafe { CStr::from_ptr(b200fft_last_error()).to_string_lossy().into_owned() }
}

/// One planned transform living on the GPU.  `Sync + Send`: the C plan handle is immutable after
/// creation and `b200fft_exec_*` may be called concurrently (same contract as every other
/// `Arc<dyn Fft<T>>`, `src/lib.rs:184`).
pub struct CudaFft<T> {
    plan: *mut B200FftPlan,
    len: usize,
    direction: FftDirection,
    _phantom: std::marker::PhantomData<T>,
}
unsafe impl<T> Send for CudaFft<T> {}
unsafe impl<T> Sync for CudaFft<T> {}

impl<T: FftNum> CudaFft<T> {
    /// `None` when `T` is neither f32 nor f64 (the AVX planner does the same TypeId test,
    /// `src/avx/avx_planner.rs:149-163`) or when the library cannot plan `len`.
    pub fn new(len: usize, direction: FftDirection, device: i32) -> Option<Self> {
        let precision = if TypeId::of::<T>() == TypeId::of::<f32>() {
            0
        } else if TypeId::of::<T>() == TypeId::of::<f64>() {
            1
        } else {
            return None;
        };
        let dir = match direction {
            FftDirection::Forward => 0,
            FftDirection::Inverse => 1,
        };
        let mut plan: *mut B200FftPlan = std::ptr::null_mut();
        let rc = unsafe { b200fft_plan_create(&mut plan, len as u64, dir, precision, device) };
        if rc != 0 {
            return None;
        }
        Some(Self { plan, len, direction, _phantom: std::marker::PhantomData })
    }
}

impl<T: FftNum> CudaFft<T> {
    /// Planning owned by Rust (north_star: "Rust host code owns planning ... and calls through a thin extern C FFI"): the
    /// recipe `FftPlannerScalar::design_fft_for_len` produced, handed over as data.  `None` when the library has no kernel
    /// sequence for that decomposition -- the caller then retries with `CudaFft::new` (the library's own choice).
    pub fn from_recipe(nodes: &[B200FftRecipeNode], direction: FftDirection, device: i32) -> Option<Self> {
        let precision = if TypeId::of::<T>() == TypeId::of::<f32>() { 0 } else if TypeId::of::<T>() == TypeId::of::<f64>() { 1 } else { return None };
        let dir = match direction {
            FftDirection::Forward => 0,
            FftDirection::Inverse => 1,
        };
        let mut plan: *mut B200FftPlan = std::ptr::null_mut();
        let rc = unsafe { b200fft_plan_create_from_recipe(&mut plan, nodes.as_ptr(), nodes.len() as u32, dir, precision, device) };
        if rc != 0 {
            return None;
        }
        Some(Self { plan, len: nodes[0].len as usize, direction, _phantom: std::marker::PhantomData })
    }
}

impl<T> Drop for CudaFft<T> {
    fn drop(&mut self) {
        unsafe { b200fft_plan_destroy(self.plan) };
    }
}

impl<T: FftNum> Fft<T> for CudaFft<T> {
    fn process_with_scratch(&self, buffer: &mut [Complex<T>], _scratch: &mut [Complex<T>]) {
        // Complex<T> is repr(C) {re, im}: the slice IS a float2/double2 array (CHANGELOG.md:139).
        let rc = unsafe { b200fft_exec_host_inplace(self.plan, buffer.as_mut_ptr() as *mut c_void, buffer.len() as u64) };
        if rc != 0 {
            // the library returns the text of common::fft_error_inplace (src/common.rs:13-39)
            panic!("{}", last_error());
        }
    }
    fn process_outofplace_with_scratch(&self, input: &mut [Complex<T>], output: &mut [Complex<T>], _scratch: &mut [Complex<T>]) {
        if input.len() != output.len() {
            crate::common::fft_error_outofplace(self.len, input.len(), output.len(), 0, 0);
        }
        let rc = unsafe {
            b200fft_exec_host_outofplace(self.plan, input.as_ptr() as *const c_void, output.as_mut_ptr() as *mut c_void, input.len() as u64)
        };
        if rc != 0 {
            panic!("{}", last_error());
        }
    }
    fn process_immutable_with_scratch(&self, input: &[Complex<T>], output: &mut [Complex<T>], _scratch: &mut [Complex<T>]) {
        if input.len() != output.len() {
            crate::common::fft_error_immut(self.len, input.len(), output.len(), 0, 0);
        }
        let rc = unsafe {
            b200fft_exec_host_outofplace(self.plan, input.as_ptr() as *const c_void, output.as_mut_ptr() as *mut c_void, input.len() as u64)
        };
        if rc != 0 {
            panic!("{}", last_error());
        }
    }
    // a backend may ask for no scratch at all (src/lib.rs:259-261)
    fn get_inplace_scratch_len(&self) -> usize {
        0
    }
    fn get_outofplace_scratch_len(&self) -> usize {
        0
    }
    fn get_immutable_scratch_len(&self) -> usize {
        0
    }
}
impl<T> Length for CudaFft<T> {
    fn len(&self) -> usize {
        self.len
    }
}
impl<T> Direction for CudaFft<T> {
    fn fft_direction(&self) -> FftDirection {
        self.direction
    }
}
