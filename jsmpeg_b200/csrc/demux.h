// demux.h -- the host side of the device demultiplexers of many requests per call (engine.cu demux_many, tsdemux.cu,
// psdemux.cu): the buffers a call reads and writes, and each format's steps.
#pragma once
#include "buffers.h"

// The per-call I/O of a demux pass: the staged request bytes, pinned room for the streams' left-over bytes on their
// way up, the request table (the host fills it, the device reads it) and the result table (the other way round), the
// call's PES list in (request, offset) order, and cub's temporary storage.  A buffer too small for a call grows to 5/4
// of what the call needs.
template <class Req, class Out>
struct DemuxIo {
	DeviceBuffer<uint8_t> stage;
	PinnedBuffer<uint8_t> h_left;
	DeviceBuffer<Req> req;
	PinnedBuffer<Req> h_req;
	DeviceBuffer<Out> out;
	PinnedBuffer<Out> h_out;
	DeviceBuffer<uint32_t> pes_offset;
	DeviceBuffer<uint64_t> pes_pts;
	PinnedBuffer<uint32_t> h_pes_offset;
	PinnedBuffer<uint64_t> h_pes_pts;
	DeviceBuffer<uint8_t> temp;

	// room for `rows` request and result rows, `staged` staging bytes and `left` left-over bytes; the staging buffer
	// keeps 32 readable bytes behind them (PS's candidate search loads 16 bytes at the last multiple of 16 and a
	// look-ahead word behind it)
	void begin(size_t rows, size_t staged, size_t left) {
		grow(stage, staged + 32);
		grow(h_left, left);
		grow(req, rows);
		grow(h_req, rows);
		grow(out, rows);
		grow(h_out, rows);
	}
	// room for a PES list of n entries
	void reserve_pes(size_t n) {
		grow(pes_offset, n);
		grow(pes_pts, n);
		grow(h_pes_offset, n);
		grow(h_pes_pts, n);
	}
	void *temp_storage(size_t bytes) {
		grow(temp, bytes);
		return temp.data();
	}
	template <class B>
	static void grow(B &buf, size_t need) {
		if (need > buf.size()) buf.reserve(need + need / 4);
	}
};

// MPEG-TS (tsdemux.cu, tsdemux.cuh).  A call: ts_call_begin makes room for n_req requests of n_slots packet slots in
// all (max_req: the most requests a call of the batch can have, which fixes the event key's width), before the caller
// uploads io.req[0 .. n_req] (entry n_req: slot0 = n_slots) with the staged bytes; ts_call_measure queues the grid,
// classify, bind and place scans and the D2H of the per-request results to io.h_out; once the caller has set every
// request's dst / es_base and uploaded the table again, ts_call_gather queues the copy of the payloads and the PES
// list.  Both return the launches they queued.
struct TsReq;
struct TsReqOut;
struct TsScratch;
using TsIo = DemuxIo<TsReq, TsReqOut>;
TsScratch *ts_scratch_create();
void ts_scratch_destroy(TsScratch *s);
void ts_call_begin(TsScratch *s, TsIo &io, uint32_t n_req, uint32_t n_slots, uint32_t max_req);
uint32_t ts_call_measure(TsScratch *s, TsIo &io, cudaStream_t st);
uint32_t ts_call_gather(TsScratch *s, TsIo &io, uint32_t pad, cudaStream_t st);

// MPEG program streams (psdemux.cu, psdemux.cuh).  A call: ps_call_begin makes room for n_req requests staged at
// 16-byte aligned offsets (`staged` bytes with the padding), before the caller uploads io.req[0 .. n_req) with the
// staged bytes; ps_call_candidates queues the candidate search and the D2H of its counts; once the caller has
// synchronised, ps_call_measure sizes the per-candidate scratch and the PES list by them, queues sort, link, doubling,
// heads, marking, classify, place scan and totals and the D2H of the per-request results to io.h_out; once the caller
// has set every request's dst / es_base and uploaded the table again, ps_call_gather queues the copy of the payloads
// and the PES list.  The three return the launches they queued.
struct PsReq;
struct PsReqOut;
struct PsScratch;
using PsIo = DemuxIo<PsReq, PsReqOut>;
PsScratch *ps_scratch_create();
void ps_scratch_destroy(PsScratch *s);
void ps_call_begin(PsScratch *s, uint32_t n_req, uint32_t staged);
uint32_t ps_call_candidates(PsScratch *s, PsIo &io, cudaStream_t st);
uint32_t ps_call_measure(PsScratch *s, PsIo &io, cudaStream_t st);
uint32_t ps_call_gather(PsScratch *s, PsIo &io, uint32_t pad, cudaStream_t st);
