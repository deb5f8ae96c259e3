//! `CudaDct<T>`: the DCT / DST plans of include/b200fft.h (`b200fft_dct_*`) in the shape of the `rustdct` crate's
//! `Dct2` / `Dct3` / `Dct4` / `Dst2` / `Dst3` / `Dst4` traits (`process_dct2(&mut buffer)` ...), which sit on RustFFT's `Fft` the
//! way `realfft` does.  Unnormalised like rustdct: DCT-III(DCT-II(x)) = (N/2) x.  NOT COMPILED IN THIS REPOSITORY (no rustc).

use std::any::TypeId;
use std::marker::PhantomData;
use std::os::raw::{c_char, c_int, c_void};

use crate::common::FftNum;

#[repr(C)]
pub struct B200FftDctPlan {
    _private: [u8; 0],
}

/// `B200FFT_DCT2` ... `B200FFT_DST4`
#[derive(Clone, Copy, Debug, PartialEq, Eq)]
#[repr(i32)]
pub enum DctKind {
    Dct2 = 0,
    Dct3 = 1,
    Dct4 = 2,
    Dst2 = 3,
    Dst3 = 4,
    Dst4 = 5,
}

#[link(name = "b200fft")]
extern "C" {
    fn b200fft_dct_plan_create(out: *mut *mut B200FftDctPlan, len: u64, kind: c_int, precision: c_int, device: c_int) -> c_int;
    fn b200fft_dct_plan_destroy(plan: *mut B200FftDctPlan) -> c_int;
    fn b200fft_dct_describe(plan: *const B200FftDctPlan, buf: *mut c_char, cap: u64) -> c_int;
    fn b200fft_dct_host(plan: *const B200FftDctPlan, input: *const c_void, output: *mut c_void, batch: u64) -> c_int;
}

/// One planned DCT / DST of one length and kind on the GPU.  `Sync + Send`: the plan handle is immutable.
pub struct CudaDct<T> {
    plan: *mut B200FftDctPlan,
    len: usize,
    kind: DctKind,
    _t: PhantomData<T>,
}
unsafe impl<T> Send for CudaDct<T> {}
unsafe impl<T> Sync for CudaDct<T> {}

impl<T: FftNum> CudaDct<T> {
    pub fn new(len: usize, kind: DctKind) -> Result<Self, String> {
        let precision = if TypeId::of::<T>() == TypeId::of::<f32>() { 0 } else if TypeId::of::<T>() == TypeId::of::<f64>() { 1 } else {
            return Err("CudaDct supports f32 and f64 only".into());
        };
        let mut plan = std::ptr::null_mut();
        let rc = unsafe { b200fft_dct_plan_create(&mut plan, len as u64, kind as c_int, precision, 0) };
        if rc != 0 {
            return Err(super::last_error_text());
        }
        Ok(Self { plan, len, kind, _t: PhantomData })
    }
    pub fn len(&self) -> usize {
        self.len
    }
    pub fn kind(&self) -> DctKind {
        self.kind
    }
    pub fn describe(&self) -> String {
        let mut buf = vec![0u8; 512];
        let n = unsafe { b200fft_dct_describe(self.plan, buf.as_mut_ptr().cast(), buf.len() as u64) };
        if n < 0 {
            return String::new();
        }
        buf.truncate(n as usize);
        String::from_utf8_lossy(&buf).into_owned()
    }
    /// Every contiguous chunk of len() samples of `buffer`, in place (rustdct's `process_dct2(&mut buffer)` and friends; its
    /// scratch variants need no scratch here).  Panics with the library's message, as rustdct panics on a bad length.
    pub fn process(&self, buffer: &mut [T]) {
        if self.len == 0 {
            return;
        }
        assert!(buffer.len() % self.len == 0, "Dct: buffer holds {} samples, expected a multiple of {}", buffer.len(), self.len);
        let rc = unsafe { b200fft_dct_host(self.plan, buffer.as_ptr().cast(), buffer.as_mut_ptr().cast(), (buffer.len() / self.len) as u64) };
        if rc != 0 {
            panic!("{}", super::last_error_text());
        }
    }
    pub fn process_dct2(&self, buffer: &mut [T]) { debug_assert_eq!(self.kind, DctKind::Dct2); self.process(buffer) }
    pub fn process_dct3(&self, buffer: &mut [T]) { debug_assert_eq!(self.kind, DctKind::Dct3); self.process(buffer) }
    pub fn process_dct4(&self, buffer: &mut [T]) { debug_assert_eq!(self.kind, DctKind::Dct4); self.process(buffer) }
    pub fn process_dst2(&self, buffer: &mut [T]) { debug_assert_eq!(self.kind, DctKind::Dst2); self.process(buffer) }
    pub fn process_dst3(&self, buffer: &mut [T]) { debug_assert_eq!(self.kind, DctKind::Dst3); self.process(buffer) }
    pub fn process_dst4(&self, buffer: &mut [T]) { debug_assert_eq!(self.kind, DctKind::Dst4); self.process(buffer) }
}

impl<T> Drop for CudaDct<T> {
    fn drop(&mut self) {
        unsafe { b200fft_dct_plan_destroy(self.plan) };
    }
}

#[repr(C)]
pub struct B200FftDctnPlan {
    _private: [u8; 0],
}

#[link(name = "b200fft")]
extern "C" {
    fn b200fft_dctn_plan_create(out: *mut *mut B200FftDctnPlan, shape: *const u64, rank: c_int, kind: c_int, precision: c_int, device: c_int) -> c_int;
    fn b200fft_dctn_plan_destroy(plan: *mut B200FftDctnPlan) -> c_int;
    fn b200fft_dctn_describe(plan: *const B200FftDctnPlan, buf: *mut c_char, cap: u64) -> c_int;
    fn b200fft_dctn_host(plan: *const B200FftDctnPlan, input: *const c_void, output: *mut c_void, batch: u64) -> c_int;
}

/// One planned 2-D or 3-D DCT / DST (`b200fft_dctn_*`): the same kind along each of the last `shape.len()` axes of contiguous
/// row-major arrays, unnormalised (= scipy.fft.dctn / dstn / 2^rank).  `Sync + Send`: the plan handle is immutable.
pub struct CudaDctNd<T> {
    plan: *mut B200FftDctnPlan,
    shape: Vec<usize>,
    kind: DctKind,
    _t: PhantomData<T>,
}
unsafe impl<T> Send for CudaDctNd<T> {}
unsafe impl<T> Sync for CudaDctNd<T> {}

impl<T: FftNum> CudaDctNd<T> {
    /// `shape`: 2 or 3 axis lengths, each one the 1-D plan of `kind` accepts.
    pub fn new(shape: &[usize], kind: DctKind) -> Result<Self, String> {
        let precision = if TypeId::of::<T>() == TypeId::of::<f32>() { 0 } else if TypeId::of::<T>() == TypeId::of::<f64>() { 1 } else {
            return Err("CudaDctNd supports f32 and f64 only".into());
        };
        let dims: Vec<u64> = shape.iter().map(|&n| n as u64).collect();
        let mut plan = std::ptr::null_mut();
        let rc = unsafe { b200fft_dctn_plan_create(&mut plan, dims.as_ptr(), dims.len() as c_int, kind as c_int, precision, 0) };
        if rc != 0 {
            return Err(super::last_error_text());
        }
        Ok(Self { plan, shape: shape.to_vec(), kind, _t: PhantomData })
    }
    pub fn shape(&self) -> &[usize] {
        &self.shape
    }
    pub fn kind(&self) -> DctKind {
        self.kind
    }
    pub fn describe(&self) -> String {
        let mut buf = vec![0u8; 1024];
        let n = unsafe { b200fft_dctn_describe(self.plan, buf.as_mut_ptr().cast(), buf.len() as u64) };
        if n < 0 {
            return String::new();
        }
        buf.truncate(n as usize);
        String::from_utf8_lossy(&buf).into_owned()
    }
    /// Every contiguous array of `shape` in `buffer`, in place.  Panics with the library's message on a bad length.
    pub fn process(&self, buffer: &mut [T]) {
        let size: usize = self.shape.iter().product();
        if size == 0 {
            return;
        }
        assert!(buffer.len() % size == 0, "DctNd: buffer holds {} samples, expected a multiple of {}", buffer.len(), size);
        let rc = unsafe { b200fft_dctn_host(self.plan, buffer.as_ptr().cast(), buffer.as_mut_ptr().cast(), (buffer.len() / size) as u64) };
        if rc != 0 {
            panic!("{}", super::last_error_text());
        }
    }
}

impl<T> Drop for CudaDctNd<T> {
    fn drop(&mut self) {
        unsafe { b200fft_dctn_plan_destroy(self.plan) };
    }
}

#[repr(C)]
pub struct B200FftMdctPlan {
    _private: [u8; 0],
}

#[link(name = "b200fft")]
extern "C" {
    fn b200fft_mdct_plan_create(out: *mut *mut B200FftMdctPlan, len: u64, window: *const c_void, signal_len: u64, precision: c_int,
                                device: c_int) -> c_int;
    fn b200fft_mdct_plan_destroy(plan: *mut B200FftMdctPlan) -> c_int;
    fn b200fft_mdct_describe(plan: *const B200FftMdctPlan, buf: *mut c_char, cap: u64) -> c_int;
    fn b200fft_mdct_frames(plan: *const B200FftMdctPlan) -> u64;
    fn b200fft_mdct_forward_host(plan: *const B200FftMdctPlan, signal: *const c_void, coefs: *mut c_void, batch: u64) -> c_int;
    fn b200fft_mdct_inverse_host(plan: *const B200FftMdctPlan, coefs: *const c_void, signal: *mut c_void, batch: u64) -> c_int;
}

/// One planned MDCT (rustdct's `Mdct`, from `plan_mdct(len, window_fn)`) over whole signal rows of `signal_len` samples.
///
/// Frame mapping: a row x is padded as xp = `len` zeros, x, zeros, and cut into `frames()` = ceil(signal_len / len) + 1 frames of
/// 2 len samples at a hop of len.  Row f of `forward`'s output (frame-major, `frames()` rows of len coefficients per signal row) is
/// rustdct's `process_mdct(&xp[f len .. f len + len], &xp[f len + len .. f len + 2 len], &mut row)`.  `inverse` is the
/// overlap-add of rustdct's `process_imdct(&row_f, ...)` over the frames, placed at f len, times 2 / len, cropped to
/// [len, len + signal_len): with a Princen-Bradley window (sine, Vorbis, KBD) `inverse(forward(x)) = x`.  The window has 2 len taps
/// (rustdct's `window_fn::sine` / `vorbis` evaluated by the caller).  `Sync + Send`: the plan handle is immutable.
pub struct CudaMdct<T> {
    plan: *mut B200FftMdctPlan,
    len: usize,
    signal_len: usize,
    frames: usize,
    _t: PhantomData<T>,
}
unsafe impl<T> Send for CudaMdct<T> {}
unsafe impl<T> Sync for CudaMdct<T> {}

impl<T: FftNum> CudaMdct<T> {
    pub fn new(len: usize, window: &[T], signal_len: usize) -> Result<Self, String> {
        let precision = if TypeId::of::<T>() == TypeId::of::<f32>() { 0 } else if TypeId::of::<T>() == TypeId::of::<f64>() { 1 } else {
            return Err("CudaMdct supports f32 and f64 only".into());
        };
        if window.len() != 2 * len {
            return Err(format!("an MDCT of len {} needs a window of {} taps (got {})", len, 2 * len, window.len()));
        }
        let mut plan = std::ptr::null_mut();
        let rc = unsafe { b200fft_mdct_plan_create(&mut plan, len as u64, window.as_ptr().cast(), signal_len as u64, precision, 0) };
        if rc != 0 {
            return Err(super::last_error_text());
        }
        let frames = unsafe { b200fft_mdct_frames(plan) } as usize;
        Ok(Self { plan, len, signal_len, frames, _t: PhantomData })
    }
    pub fn len(&self) -> usize {
        self.len
    }
    pub fn frames(&self) -> usize {
        self.frames
    }
    pub fn describe(&self) -> String {
        let mut buf = vec![0u8; 512];
        let n = unsafe { b200fft_mdct_describe(self.plan, buf.as_mut_ptr().cast(), buf.len() as u64) };
        if n < 0 {
            return String::new();
        }
        buf.truncate(n as usize);
        String::from_utf8_lossy(&buf).into_owned()
    }
    /// Every row of `signal` (batch * signal_len samples) into `coefs` (batch * frames() * len()).  Panics with the library's message.
    pub fn forward(&self, signal: &[T], coefs: &mut [T]) {
        assert!(signal.len() % self.signal_len == 0, "Mdct: signal holds {} samples, expected a multiple of {}", signal.len(), self.signal_len);
        let batch = signal.len() / self.signal_len;
        assert_eq!(coefs.len(), batch * self.frames * self.len, "Mdct: coefficient buffer of the wrong size");
        let rc = unsafe { b200fft_mdct_forward_host(self.plan, signal.as_ptr().cast(), coefs.as_mut_ptr().cast(), batch as u64) };
        if rc != 0 {
            panic!("{}", super::last_error_text());
        }
    }
    /// Every row of `coefs` (batch * frames() * len()) into `signal` (batch * signal_len samples).  Panics with the library's message.
    pub fn inverse(&self, coefs: &[T], signal: &mut [T]) {
        let per = self.frames * self.len;
        assert!(coefs.len() % per == 0, "Mdct: coefficient buffer holds {} values, expected a multiple of {}", coefs.len(), per);
        let batch = coefs.len() / per;
        assert_eq!(signal.len(), batch * self.signal_len, "Mdct: signal buffer of the wrong size");
        let rc = unsafe { b200fft_mdct_inverse_host(self.plan, coefs.as_ptr().cast(), signal.as_mut_ptr().cast(), batch as u64) };
        if rc != 0 {
            panic!("{}", super::last_error_text());
        }
    }
}

impl<T> Drop for CudaMdct<T> {
    fn drop(&mut self) {
        unsafe { b200fft_mdct_plan_destroy(self.plan) };
    }
}
