//go:build cuda

// decode_cuda.go -- drop-in replacement for rtlamr's protocol/decode.go that runs the Decoder hot
// path (magnitude, matched filter, quantize, pack, preamble search, slice, CRC screen) on an H100
// through libertgpu.so (include/ertgpu.h).
//
// How to use it (see INTEGRATION.md):
//   1. copy this file to <rtlamr>/protocol/decode_cuda.go
//   2. add `//go:build !cuda` as the first line of <rtlamr>/protocol/decode.go
//   3. go build -tags cuda ./...   (CGO_CFLAGS/CGO_LDFLAGS pointing at include/ and libertgpu.so)
//
// Everything exported by decode.go keeps its name, signature and meaning: PacketConfig, Decoder
// (with its Cfg field), NewDecoder, RegisterProtocol, Allocate, Decode, Log, NextPowerOf2,
// Demodulator, MagLUT, NewMagLUT.  protocol/parse.go and every parser package stay untouched,
// except r900 which reads its payload digits through Decoder.R900Digits (three-line patch in
// INTEGRATION.md) because its DSP half also moved to the GPU.
//
// STATUS: EXPERIMENTAL.  Written without a Go toolchain at hand (none in the build image): this file has
// never been compiled; parity_test.go next to it is the first thing to run where Go and an H100 exist.
// The C++ mirror in rtlamr_b200/host/ exercises the same call sequence in the parity tests.
//
// Two things a maintainer must know:
//   * input memory: `input` is an ordinary Go slice (pageable).  ertgpu_decode stages pageable memory through
//     pinned buffers owned by the handle (copy threads + chunked H2D), so the call is correct and reasonably
//     fast for large calls (bench.py reports `e2e.pageable_input_value` next to the pinned figure), but one
//     BlockSize2 (8-16 KiB) block per call, as main.go:166-186 reads them, pays a whole GPU pipeline and a
//     synchronisation per block: feed K blocks per Decode (INTEGRATION.md 1, step 5) for throughput.
//   * K > 1 and main.go's dedup: messages come back grouped per reference block and in block order, but the
//     caller's `prev/next` digest maps (main.go:251-260) are swapped once per Decode CALL, so with K blocks per
//     call a message repeated in the two blocks it straddles is suppressed inside the call only if the caller
//     swaps the maps per block.  The channel carries no block index (protocol.Message has none): use K = 1 when
//     main.go's exact dedup semantics matter, or take the C++ BlockDedup (rtlamr_b200/host/receiver.cpp), which
//     swaps per block, as the model.
package protocol

/*
#cgo CFLAGS: -I${SRCDIR}/../../include
#cgo LDFLAGS: -L${SRCDIR}/../../rtlamr_b200 -lertgpu -Wl,-rpath,${SRCDIR}/../../rtlamr_b200
#include <stdlib.h>
#include <string.h>
#include "ertgpu.h"
*/
import "C"

import (
	"fmt"
	"log"
	"math"
	"os"
	"strconv"
	"strings"
	"sync"
	"unsafe"
)

// PacketConfig specifies packet-specific radio configuration (unchanged, decode.go:27-42).
type PacketConfig struct {
	Protocol string
	Preamble string

	DataRate int

	BlockSize, BlockSize2    int
	ChipLength, SymbolLength int
	SampleRate               int

	PreambleSymbols, PacketSymbols int
	PreambleLength, PacketLength   int

	BufferLength int
	CenterFreq   uint32
}

// Decoder keeps the reference's exported surface.  Signal and Quantized stay as fields for source
// compatibility but are not maintained per block (they live in HBM); use Tap for parity checks.
type Decoder struct {
	Cfg PacketConfig
	wg  *sync.WaitGroup

	Signal    []float32
	Quantized []byte

	preambleStrs map[string]bool
	preambles    [][]Parser // per distinct preamble, in registration order
	preambleKeys []string
	protocols    []string

	h     *C.ertgpu_handle
	cands []C.ertgpu_candidate

	// digits of the candidates of the block being parsed, keyed by Data.Idx (for r900)
	digits map[int][]byte
}

func NewDecoder() Decoder {
	d := Decoder{
		wg:           new(sync.WaitGroup),
		preambleStrs: make(map[string]bool),
	}
	if rc := C.ertgpu_create(&d.h); rc != C.ERTGPU_OK {
		panic("ertgpu_create failed")
	}
	return d
}

func (d Decoder) Log() {
	log.Println("CenterFreq:", d.Cfg.CenterFreq)
	log.Println("SampleRate:", d.Cfg.SampleRate)
	log.Println("DataRate:", d.Cfg.DataRate)
	log.Println("ChipLength:", d.Cfg.ChipLength)
	log.Println("PreambleSymbols:", d.Cfg.PreambleSymbols)
	log.Println("PreambleLength:", d.Cfg.PreambleLength)
	log.Println("PacketSymbols:", d.Cfg.PacketSymbols)
	log.Println("PacketLength:", d.Cfg.PacketLength)
	log.Println("Protocols:", strings.Join(d.protocols, ","))
	log.Println("Preambles:", strings.Join(d.preambleKeys, ","))
}

func (d *Decoder) fail(what string, rc C.int) {
	panic(fmt.Sprintf("%s: libertgpu error %d: %s", what, int(rc), C.GoString(C.ertgpu_last_error(d.h))))
}

// RegisterProtocol merges the parser's config exactly like decode.go:100-128 and tells the GPU
// library about the parser's preamble, geometry and integrity screen.
func (d *Decoder) RegisterProtocol(p Parser) {
	p.SetDecoder(d)
	cfg := p.Cfg()

	d.Cfg.CenterFreq = cfg.CenterFreq
	d.Cfg.DataRate = max(d.Cfg.DataRate, cfg.DataRate)
	d.Cfg.ChipLength = max(d.Cfg.ChipLength, cfg.ChipLength)
	d.Cfg.PreambleSymbols = max(d.Cfg.PreambleSymbols, cfg.PreambleSymbols)
	d.Cfg.PacketSymbols = max(d.Cfg.PacketSymbols, cfg.PacketSymbols)

	// Start from the stock screen of the protocol name (CRC ranges etc.); unknown parsers get no
	// GPU screen, i.e. every candidate is handed to them.
	var ep C.ertgpu_protocol
	name := C.CString(cfg.Protocol)
	defer C.free(unsafe.Pointer(name))
	if rc := C.ertgpu_stock_protocol(name, C.int32_t(cfg.ChipLength), &ep); rc != C.ERTGPU_OK {
		C.memset(unsafe.Pointer(&ep), 0, C.sizeof_ertgpu_protocol)
		ep.check_kind = C.ERTGPU_CHECK_NONE
		copyCString(unsafe.Pointer(&ep.name[0]), len(ep.name), cfg.Protocol)
	}
	copyCString(unsafe.Pointer(&ep.preamble[0]), len(ep.preamble), cfg.Preamble)
	ep.data_rate = C.int32_t(cfg.DataRate)
	ep.chip_length = C.int32_t(cfg.ChipLength)
	ep.preamble_symbols = C.int32_t(cfg.PreambleSymbols)
	ep.packet_symbols = C.int32_t(cfg.PacketSymbols)
	ep.center_freq = C.uint32_t(cfg.CenterFreq)
	if rc := C.ertgpu_register_protocol(d.h, &ep); rc != C.ERTGPU_OK {
		d.fail("RegisterProtocol", rc)
	}

	d.preambleStrs[cfg.Preamble] = true
	idx := -1
	for i, k := range d.preambleKeys {
		if k == cfg.Preamble {
			idx = i
		}
	}
	if idx < 0 {
		d.preambleKeys = append(d.preambleKeys, cfg.Preamble)
		d.preambles = append(d.preambles, nil)
		idx = len(d.preambleKeys) - 1
	}
	d.preambles[idx] = append(d.preambles[idx], p)
	d.protocols = append(d.protocols, cfg.Protocol)
}

func copyCString(dst unsafe.Pointer, cap int, s string) {
	b := unsafe.Slice((*byte)(dst), cap)
	n := copy(b[:cap-1], s)
	b[n] = 0
}

// Allocate derives the lengths (decode.go:131-141) and allocates the device buffers.
// ERTGPU_DEVICE and ERTGPU_MAX_BLOCKS tune the device ordinal and the largest Decode call.
func (d *Decoder) Allocate() {
	device, _ := strconv.Atoi(os.Getenv("ERTGPU_DEVICE"))
	maxBlocks, _ := strconv.ParseInt(os.Getenv("ERTGPU_MAX_BLOCKS"), 10, 64)
	if rc := C.ertgpu_allocate(d.h, C.int32_t(device), C.int64_t(maxBlocks), 0); rc != C.ERTGPU_OK {
		d.fail("Allocate", rc)
	}
	var c C.ertgpu_decoder_config
	C.ertgpu_get_config(d.h, &c)
	d.Cfg.SymbolLength = int(c.symbol_length)
	d.Cfg.SampleRate = int(c.sample_rate)
	d.Cfg.PreambleLength = int(c.preamble_length)
	d.Cfg.PacketLength = int(c.packet_length)
	d.Cfg.BlockSize = int(c.block_size)
	d.Cfg.BlockSize2 = int(c.block_size2)
	d.Cfg.BufferLength = int(c.buffer_length)

	d.Signal = make([]float32, d.Cfg.BlockSize+d.Cfg.SymbolLength)
	d.Quantized = make([]byte, d.Cfg.BufferLength)
	d.cands = make([]C.ertgpu_candidate, 4096)
}

// Decode accepts one OR MORE whole sample blocks (len(input) = N*BlockSize2) and returns a channel
// of messages, equivalent to N sequential reference Decode calls (decode.go:163-197).
func (d *Decoder) Decode(input []byte) chan Message {
	if len(input) == 0 || len(input)%d.Cfg.BlockSize2 != 0 {
		// the reference indexes past the slice and panics (decode.go:222)
		panic(fmt.Sprintf("protocol: Decode needs whole blocks of %d bytes, got %d", d.Cfg.BlockSize2, len(input)))
	}
	var n C.size_t
	rc := C.ertgpu_decode(d.h, (*C.uint8_t)(unsafe.Pointer(&input[0])), C.size_t(len(input)),
		C.ERTGPU_DECODE_ONLY_VALID, &d.cands[0], C.size_t(len(d.cands)), &n)
	if rc == C.ERTGPU_ECAPACITY && int(n) > len(d.cands) {
		d.cands = make([]C.ertgpu_candidate, int(n))
		rc = C.ertgpu_fetch(d.h, &d.cands[0], C.size_t(len(d.cands)), &n)
	}
	if rc != C.ERTGPU_OK {
		d.fail("Decode", rc)
	}

	msgCh := make(chan Message)
	nbytes := (d.Cfg.PacketSymbols + 7) >> 3
	cands := d.cands[:int(n)]

	go func() {
		// Candidates arrive sorted by (block, preamble, idx): rebuild the reference's per-block,
		// per-preamble []Data (decode.go:177-187) and run that preamble's parsers on it.
		for i := 0; i < len(cands); {
			j := i
			var pkts []Data
			digits := make(map[int][]byte)
			for j < len(cands) && cands[j].block == cands[i].block && cands[j].preamble_id == cands[i].preamble_id {
				c := &cands[j]
				data := NewData(C.GoBytes(unsafe.Pointer(&c.bytes[0]), C.int(nbytes)))
				data.Idx = int(c.idx)
				pkts = append(pkts, data)
				if c.flags&C.ERTGPU_CAND_HAS_R900 != 0 {
					digits[data.Idx] = C.GoBytes(unsafe.Pointer(&c.r900_digits[0]), C.ERTGPU_R900_DIGITS)
				}
				j++
			}
			d.digits = digits
			parsers := d.preambles[int(cands[i].preamble_id)]
			d.wg.Add(len(parsers))
			for _, p := range parsers {
				go p.Parse(pkts, msgCh, d.wg)
			}
			d.wg.Wait() // blocks are parsed one after another, like successive Decode calls
			i = j
		}
		close(msgCh)
	}()

	return msgCh
}

// R900Digits returns the 42 base-6 payload digits the reference r900 parser would read from its
// own quantized buffer at payloadIdx + k*4*ChipLength (r900/r900.go:187-193) for the candidate
// with the given Data.Idx of the block being parsed.
func (d *Decoder) R900Digits(idx int) ([]byte, bool) {
	v, ok := d.digits[idx]
	return v, ok
}

// Tap returns the reference buffer `which` (an ERTGPU_TAP constant) as it would be after the Decode of
// `block` (parity checks only).
func (d *Decoder) Tap(which int, block int64) []byte {
	var n C.size_t
	if rc := C.ertgpu_tap(d.h, C.int32_t(which), C.int64_t(block), nil, 0, &n); rc != C.ERTGPU_OK {
		d.fail("Tap", rc)
	}
	buf := make([]byte, int(n))
	if rc := C.ertgpu_tap(d.h, C.int32_t(which), C.int64_t(block), unsafe.Pointer(&buf[0]), n, &n); rc != C.ERTGPU_OK {
		d.fail("Tap", rc)
	}
	return buf
}

// Close releases the device buffers (the reference Decoder has no Close; optional).
func (d *Decoder) Close() {
	C.ertgpu_destroy(d.h)
	d.h = nil
}

func max(a, b int) int {
	if a > b {
		return a
	}
	return b
}

// A Demodulator knows how to demodulate an array of uint8 IQ samples into an array of float32
// samples.  Kept for source compatibility (decode.go:199-225); the GPU path does not use it.
type Demodulator interface {
	Execute([]byte, []float32)
}

type MagLUT []float32

// NewMagLUT builds the 256-entry squared-magnitude table of decode.go:209-216 (host copy; the
// kernels keep their own, computed with the same float32 operations).
func NewMagLUT() MagLUT {
	table := make(MagLUT, 256)
	for v := 0; v < 256; v++ {
		x := (127.5 - float32(v)) / 127.5
		table[v] = x * x
	}
	return table
}

// Execute keeps the Demodulator contract: out[k] = lut[I_k] + lut[Q_k] (decode.go:219-225).
func (lut MagLUT) Execute(iq []byte, out []float32) {
	for k := range out {
		out[k] = lut[iq[2*k]] + lut[iq[2*k+1]]
	}
}

func NextPowerOf2(v int) int {
	return 1 << uint(math.Ceil(math.Log2(float64(v))))
}
