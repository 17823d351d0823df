// buffers.h -- owning device and pinned host allocations of the host side (engine.cu, tsdemux.cu, psdemux.cu).
//
// DeviceBuffer<T> (cudaMalloc) and PinnedBuffer<T> (cudaHostAlloc) own one allocation each and free it when they are
// reset, reassigned or destroyed.  They are move-only.  reserve(n) grows only and discards the contents: no copy, so
// a caller that keeps bytes across a regrow (the ES mirror) copies them itself.  Release uses the synchronizing
// cudaFree / cudaFreeHost, never a stream-ordered free: regrow paths rely on work still queued on a stream having
// finished with the old allocation.  Release never throws and ignores errors (a dead decoder is destroyed while its
// context may be the thing that failed), and an empty buffer makes no CUDA call at all.
#pragma once
#include <algorithm>
#include <cstddef>
#include <utility>

#include "common.cuh"

struct DeviceAlloc {
	static void *alloc(size_t bytes) {
		void *p = nullptr;
		CUDA_CHECK(cudaMalloc(&p, bytes));
		return p;
	}
	static void release(void *p) { (void)cudaFree(p); }
};

struct PinnedAlloc {
	static void *alloc(size_t bytes) {
		void *p = nullptr;
		CUDA_CHECK(cudaHostAlloc(&p, bytes, cudaHostAllocDefault));
		return p;
	}
	static void release(void *p) { (void)cudaFreeHost(p); }
};

template <typename T, typename Alloc>
class Buffer {
public:
	Buffer() = default;
	explicit Buffer(size_t n) { reserve(n); }
	Buffer(Buffer &&o) noexcept : p_(std::exchange(o.p_, nullptr)), n_(std::exchange(o.n_, 0)) {}
	Buffer &operator=(Buffer &&o) noexcept {
		if (this != &o) {
			reset();
			p_ = std::exchange(o.p_, nullptr);
			n_ = std::exchange(o.n_, 0);
		}
		return *this;
	}
	Buffer(const Buffer &) = delete;
	Buffer &operator=(const Buffer &) = delete;
	~Buffer() { reset(); }

	T *data() const { return p_; }  // nullptr while empty
	size_t size() const { return n_; }  // elements
	T &operator[](size_t i) const { return p_[i]; }

	// Room for n elements: a new allocation of max(n, 1) elements unless this one already has room.  The old
	// contents are gone either way when it reallocates.  Returns whether it did.
	bool reserve(size_t n) {
		if (p_ && n <= n_) return false;
		reset();
		p_ = static_cast<T *>(Alloc::alloc(std::max<size_t>(n, 1) * sizeof(T)));
		n_ = n;
		return true;
	}

	void reset() noexcept {
		if (p_) Alloc::release(p_);
		p_ = nullptr;
		n_ = 0;
	}

private:
	T *p_ = nullptr;
	size_t n_ = 0;
};

template <typename T>
using DeviceBuffer = Buffer<T, DeviceAlloc>;
template <typename T>
using PinnedBuffer = Buffer<T, PinnedAlloc>;
