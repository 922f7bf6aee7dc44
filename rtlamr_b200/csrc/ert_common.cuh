// ert_common.cuh -- device-side configuration shared by the libertgpu kernels.
//
// Geometry names follow protocol.PacketConfig (reference protocol/decode.go:27-42):
// CL=ChipLength, SL=SymbolLength, BS=BlockSize, PS/PK=Preamble/PacketSymbols,
// PL/PKL=Preamble/PacketLength, BUF=BufferLength.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/ertgpu.h"

namespace ert {

struct DevProto {
    int32_t preamble_id;
    int32_t check_kind;
    int32_t packet_bytes;  // this parser's own (PacketSymbols+7)>>3
    int32_t crc_from, crc_to;
    uint16_t crc_init, crc_residue;
    int32_t table;  // index into the CRC table array
};

struct DevCfg {
    int32_t CL, SL, BS, PS, PK, PL, PKL, BUF;
    int32_t words_per_block;  // BS/32
    int32_t hist_words;       // ceil(PKL/32): bit-plane history kept in front of a call's bits
    int32_t hist_samples;     // IQ history kept in front of a call's samples (= PKL)
    int32_t packet_bytes;     // (PK+7)>>3
    int32_t npre;
    int32_t pre_nbits[ERTGPU_MAX_PROTOCOLS];
    uint8_t pre_bits[ERTGPU_MAX_PROTOCOLS][ERTGPU_MAX_PREAMBLE];
    int32_t pre_has_r900[ERTGPU_MAX_PROTOCOLS];
    int32_t nproto;
    DevProto proto[ERTGPU_MAX_PROTOCOLS];
};

// BlockSize is a power of two (decode.go:138, NextPowerOf2): block = s >> bs_shift, idx = s & (BS-1)
__device__ __forceinline__ int bs_shift(const DevCfg& c) { return 31 - __clz(c.BS); }

// A search hit before slicing: start position (in samples) relative to
// (first global sample of the call) - PKL, and the preamble that matched.
struct RawHit {
    unsigned long long s;
    int32_t preamble_id;
    int32_t pad;
};

// One word of 32 consecutive start positions with at least one hit: what Search hands to Slice.
// Start gw*32 + k (k counted from the MSB of `mask`) is a hit iff bit 31-k of mask is set; its RawHit
// (and, for r900, its payload digits) sits at index slot + (number of set bits above it).
struct HitWord {
    unsigned long long gw;    // call-relative word of starts
    unsigned long long slot;  // index of the word's first RawHit
    uint32_t mask;
    int32_t preamble_id;
};

// counters of one pipeline (unsigned long long each)
enum { kCntHits = 0, kCntOut = 1, kCntValid = 2, kCntTile = 3, kCntWords = 4, kCntN = 8 };

// Programmatic dependent launch (sm_90+): a kernel launched with the programmaticStreamSerialization attribute may
// become resident while the kernel in front of it on the stream is still running; pdl_wait() blocks until that
// kernel has completed and its writes are visible (a no-op for an ordinary launch), pdl_launch_dependents() tells
// the scheduler that the NEXT kernel's CTAs may be brought in as soon as there is room.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

}  // namespace ert
