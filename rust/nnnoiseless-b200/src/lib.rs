//! Drop-in for the denoise path of `nnnoiseless` (`DenoiseState`, `RnnModel`) backed by the H100 CUDA
//! library through the C ABI of `include/rnnoise.h`.  UNVERIFIED: no Rust toolchain exists in the build
//! image; signatures follow `src/denoise.rs:44-116` and `src/rnn.rs:72-94` of the reference.
use std::marker::PhantomData;
use std::os::raw::{c_float, c_int, c_long, c_uchar, c_void};

#[repr(C)] pub struct RawState { _p: [u8; 0] }
#[repr(C)] pub struct RawModel { _p: [u8; 0] }
#[repr(C)] pub struct RawBatch { _p: [u8; 0] }

extern "C" {
    fn rnnoise_create(model: *mut RawModel) -> *mut RawState;
    fn rnnoise_destroy(st: *mut RawState);
    fn rnnoise_process_frame(st: *mut RawState, out: *mut c_float, input: *mut c_float) -> c_float;
    fn rnnoise_model_from_bytes(bytes: *const c_uchar, len: usize) -> *mut RawModel;
    fn rnnoise_model_free(model: *mut RawModel);
    fn rnnoise_batch_create(model: *const RawModel, n_streams: c_int, device: c_int) -> *mut RawBatch;
    fn rnnoise_batch_destroy(b: *mut RawBatch);
    fn rnnoise_batch_process_host(b: *mut RawBatch, out: *mut c_float, input: *const c_float, vad: *mut c_float, n_frames: c_int) -> c_int;
    fn rnnoise_batch_process_device(b: *mut RawBatch, out: *mut c_float, input: *const c_float, vad: *mut c_float, n_frames: c_int,
                                    stream_stride: c_long, frame_stride: c_long, cuda_stream: *mut c_void) -> c_int;
    fn rnnoise_batch_process_streams_host(b: *mut RawBatch, streams: *const c_int, n: c_int, out: *mut c_float, input: *const c_float,
                                          vad: *mut c_float, n_frames: c_int) -> c_int;
    fn rnnoise_batch_process_streams_device(b: *mut RawBatch, streams: *const c_int, n: c_int, out: *mut c_void, input: *const c_void,
                                            pcm16: c_int, vad: *mut c_float, n_frames: c_int, stream_stride: c_long,
                                            sample_stride: c_long, frame_stride: c_long, cuda_stream: *mut c_void) -> c_int;
    fn rnnoise_batch_add_model(b: *mut RawBatch, model: *const RawModel) -> c_int;
    fn rnnoise_batch_set_stream_models(b: *mut RawBatch, streams: *const c_int, n: c_int, model_ids: *const c_int) -> c_int;
    fn rnnoise_batch_get_stream_models(b: *const RawBatch, streams: *const c_int, n: c_int, model_ids: *mut c_int) -> c_int;
}

pub const FRAME_SIZE: usize = 480;

/// `RnnModel` (src/rnn.rs:55-62).
pub struct RnnModel { raw: *mut RawModel }
unsafe impl Send for RnnModel {}
unsafe impl Sync for RnnModel {}

impl RnnModel {
    /// `RnnModel::from_bytes` (src/rnn.rs:75): `None` for malformed bytes.
    pub fn from_bytes(bytes: &[u8]) -> Option<RnnModel> {
        let raw = unsafe { rnnoise_model_from_bytes(bytes.as_ptr(), bytes.len()) };
        if raw.is_null() { None } else { Some(RnnModel { raw }) }
    }
    /// `RnnModel::from_static_bytes` (src/rnn.rs:92): the C library copies the bytes, so this is an alias.
    pub fn from_static_bytes(bytes: &'static [u8]) -> Option<RnnModel> { Self::from_bytes(bytes) }
}
impl Drop for RnnModel { fn drop(&mut self) { unsafe { rnnoise_model_free(self.raw) } } }

/// `DenoiseState<'model>` (src/denoise.rs:37-42).  The built-in model is selected with `new()`.
pub struct DenoiseState<'model> { raw: *mut RawState, _model: PhantomData<&'model RnnModel> }
unsafe impl<'m> Send for DenoiseState<'m> {}
unsafe impl<'m> Sync for DenoiseState<'m> {}

impl DenoiseState<'static> {
    pub const FRAME_SIZE: usize = FRAME_SIZE;
    /// `DenoiseState::new()` (src/denoise.rs:53).  Panics if no CUDA device is usable (there is no CPU fallback).
    pub fn new() -> Box<DenoiseState<'static>> {
        let raw = unsafe { rnnoise_create(std::ptr::null_mut()) };
        assert!(!raw.is_null(), "rnnoise_create failed (no CUDA device?)");
        Box::new(DenoiseState { raw, _model: PhantomData })
    }
}
impl<'model> DenoiseState<'model> {
    /// `DenoiseState::with_model(&model)` (src/denoise.rs:72): the model is borrowed and must outlive the state.
    pub fn with_model(model: &'model RnnModel) -> Box<DenoiseState<'model>> {
        let raw = unsafe { rnnoise_create(model.raw) };
        assert!(!raw.is_null(), "rnnoise_create failed (no CUDA device?)");
        Box::new(DenoiseState { raw, _model: PhantomData })
    }
    /// `process_frame(&mut self, output, input) -> f32` (src/denoise.rs:95): both slices must hold 480 samples.
    pub fn process_frame(&mut self, output: &mut [f32], input: &[f32]) -> f32 {
        assert!(input.len() == FRAME_SIZE && output.len() == FRAME_SIZE);
        output.copy_from_slice(input);
        unsafe { rnnoise_process_frame(self.raw, output.as_mut_ptr(), output.as_mut_ptr()) }
    }
}
impl<'m> Drop for DenoiseState<'m> { fn drop(&mut self) { unsafe { rnnoise_destroy(self.raw) } } }

/// N independent `DenoiseState`s advanced together on one GPU (additive API).
pub struct DenoiseBatch { raw: *mut RawBatch, n_streams: usize }
unsafe impl Send for DenoiseBatch {}

impl DenoiseBatch {
    pub fn new(n_streams: usize, model: Option<&RnnModel>, device: i32) -> Option<DenoiseBatch> {
        let m = model.map_or(std::ptr::null(), |m| m.raw as *const RawModel);
        let raw = unsafe { rnnoise_batch_create(m, n_streams as c_int, device as c_int) };
        if raw.is_null() { None } else { Some(DenoiseBatch { raw, n_streams }) }
    }
    /// Host buffers laid out `[n_frames][n_streams][480]`; `vad` (optional) `[n_frames][n_streams]`.
    pub fn process_frames(&mut self, output: &mut [f32], input: &[f32], vad: Option<&mut [f32]>, n_frames: usize) -> Result<(), ()> {
        assert!(input.len() == n_frames * self.n_streams * FRAME_SIZE && output.len() == input.len());
        let v = vad.map_or(std::ptr::null_mut(), |v| { assert!(v.len() == n_frames * self.n_streams); v.as_mut_ptr() });
        let rc = unsafe { rnnoise_batch_process_host(self.raw, output.as_mut_ptr(), input.as_ptr(), v, n_frames as c_int) };
        if rc == 0 { Ok(()) } else { Err(()) }
    }
    /// Device buffers (raw CUDA pointers), strides in samples; asynchronous on `cuda_stream` when it is non-null.
    pub unsafe fn process_frames_device(&mut self, output: *mut f32, input: *const f32, vad: *mut f32, n_frames: usize,
                                        stream_stride: i64, frame_stride: i64, cuda_stream: *mut c_void) -> Result<(), ()> {
        let rc = rnnoise_batch_process_device(self.raw, output, input, vad, n_frames as c_int, stream_stride as c_long,
                                              frame_stride as c_long, cuda_stream);
        if rc == 0 { Ok(()) } else { Err(()) }
    }
    /// Advance only the listed streams (distinct indices, any order) by `n_frames`; the other streams are not touched.
    /// Host buffers laid out `[n_frames][streams.len()][480]`, row r belonging to `streams[r]`; `vad` (optional)
    /// `[n_frames][streams.len()]`.  The indices are checked by the library: a bad list is an `Err` and changes nothing.
    pub fn process_streams(&mut self, streams: &[i32], output: &mut [f32], input: &[f32], vad: Option<&mut [f32]>,
                           n_frames: usize) -> Result<(), ()> {
        let n = streams.len();
        assert!(input.len() == n_frames * n * FRAME_SIZE && output.len() == input.len());
        let v = vad.map_or(std::ptr::null_mut(), |v| { assert!(v.len() == n_frames * n); v.as_mut_ptr() });
        let rc = unsafe {
            rnnoise_batch_process_streams_host(self.raw, streams.as_ptr(), n as c_int, output.as_mut_ptr(), input.as_ptr(), v,
                                               n_frames as c_int)
        };
        if rc == 0 { Ok(()) } else { Err(()) }
    }
    /// Device buffers (raw CUDA pointers) of the listed streams, float samples, element strides; asynchronous on
    /// `cuda_stream` when it is non-null.
    pub unsafe fn process_streams_device(&mut self, streams: &[i32], output: *mut f32, input: *const f32, vad: *mut f32,
                                         n_frames: usize, stream_stride: i64, frame_stride: i64,
                                         cuda_stream: *mut c_void) -> Result<(), ()> {
        let rc = rnnoise_batch_process_streams_device(self.raw, streams.as_ptr(), streams.len() as c_int, output as *mut c_void,
                                                      input as *const c_void, 0, vad, n_frames as c_int, stream_stride as c_long,
                                                      1, frame_stride as c_long, cuda_stream);
        if rc == 0 { Ok(()) } else { Err(()) }
    }
    /// Add a model of this batch's geometry to its model table (the weights are copied); returns its index, the batch's
    /// own model being 0.  A model of another geometry is an `Err`.
    pub fn add_model(&mut self, model: &RnnModel) -> Result<usize, ()> {
        let k = unsafe { rnnoise_batch_add_model(self.raw, model.raw) };
        if k >= 0 { Ok(k as usize) } else { Err(()) }
    }
    /// Stream `streams[r]` runs on model `model_ids[r]` from the next frame on; the streams keep their state.  Every index
    /// and id is checked first: a bad one is an `Err` and changes nothing.
    pub fn set_stream_models(&mut self, streams: &[i32], model_ids: &[i32]) -> Result<(), ()> {
        assert!(streams.len() == model_ids.len());
        let rc = unsafe { rnnoise_batch_set_stream_models(self.raw, streams.as_ptr(), streams.len() as c_int, model_ids.as_ptr()) };
        if rc == 0 { Ok(()) } else { Err(()) }
    }
    /// The model index of each listed stream.
    pub fn stream_models(&self, streams: &[i32]) -> Result<Vec<i32>, ()> {
        let mut ids = vec![0i32; streams.len()];
        let rc = unsafe { rnnoise_batch_get_stream_models(self.raw, streams.as_ptr(), streams.len() as c_int, ids.as_mut_ptr()) };
        if rc == 0 { Ok(ids) } else { Err(()) }
    }
}
impl Drop for DenoiseBatch { fn drop(&mut self) { unsafe { rnnoise_batch_destroy(self.raw) } } }
