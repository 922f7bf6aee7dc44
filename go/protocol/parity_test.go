//go:build cuda

// parity_test.go -- the cuda-tag Decoder against golden vectors dumped by the STOCK Go decoder.
//
// 1. On any Go machine, produce the dump with the unmodified reference (go/goldengen/README.md):
//      GOLDEN_IN=assets/sample.bin GOLDEN_OUT=go_dump_sample_cl78_scm.jsonl GOLDEN_MSGTYPES=scm GOLDEN_CL=78 \
//        go test ./protocol -run TestDumpGolden -count=1            (build WITHOUT -tags cuda)
// 2. On an H100 machine, with decode_cuda.go in place:
//      ERT_GOLDEN=go_dump_sample_cl78_scm.jsonl ERT_GOLDEN_IN=assets/sample.bin \
//        go test -tags cuda ./protocol -run TestCudaParity -count=1
//
// Checks, block by block (every block is its own Decode call, like main.go:235): the candidate list
// (preamble, Idx, Bytes) equals the stock decoder's where the stock Search is exact (SymbolLength % 8 == 0;
// for other chip lengths the stock byte pre-filter drops candidates, decode.go:256,271, and the stock list must
// be a SUBSET), and the Quantized / packed / Signal / csum taps are bit-identical at the dumped blocks.
//
// Written without a Go toolchain at hand; compiled and run only where Go and an H100 exist.
package protocol

import (
	"bufio"
	"bytes"
	"encoding/hex"
	"encoding/json"
	"os"
	"sync"
	"testing"
)

type goldenLine struct {
	Kind      string   `json:"kind"`
	Block     int      `json:"block"`
	Preamble  string   `json:"preamble"`
	Idx       int      `json:"idx"`
	Bytes     string   `json:"bytes"`
	Signal    string   `json:"signal"`
	Csum      string   `json:"csum"`
	Quantized string   `json:"quantized"`
	Packed    string   `json:"packed"`
	Msgtypes  []string `json:"msgtypes"`
	ChipLen   int      `json:"chip_length"`
}

type parityParser struct {
	cfg   PacketConfig
	mu    *sync.Mutex
	block *int
	got   map[[3]string]bool // (block, preamble, idx|bytes)
}

func (p parityParser) SetDecoder(*Decoder) {}
func (p parityParser) Cfg() PacketConfig   { return p.cfg }
func (p parityParser) Parse(pkts []Data, msgCh chan Message, wg *sync.WaitGroup) {
	p.mu.Lock()
	for _, pkt := range pkts {
		p.got[[3]string{itoa(*p.block), p.cfg.Preamble, itoa(pkt.Idx) + ":" + hex.EncodeToString(pkt.Bytes)}] = true
	}
	p.mu.Unlock()
	wg.Done()
}

func itoa(v int) string {
	b, _ := json.Marshal(v)
	return string(b)
}

func stockConfig(name string, chipLength int) PacketConfig {
	c := PacketConfig{Protocol: name, CenterFreq: 912600155, DataRate: 32768, ChipLength: chipLength}
	switch name {
	case "scm":
		c.Preamble, c.PreambleSymbols, c.PacketSymbols = "111110010101001100000", 21, 96
	case "scm+":
		c.Preamble, c.PreambleSymbols, c.PacketSymbols = "0001011010100011", 16, 128
	case "idm", "netidm":
		c.Preamble, c.PreambleSymbols, c.PacketSymbols = "01010101010101010001011010100011", 32, 92*8
	case "r900", "r900bcd":
		c.Preamble, c.PreambleSymbols, c.PacketSymbols = "00000000000000001110010101100100", 32, 116
		c.CenterFreq = 912380000
	}
	return c
}

func TestCudaParity(t *testing.T) {
	dump, in := os.Getenv("ERT_GOLDEN"), os.Getenv("ERT_GOLDEN_IN")
	if dump == "" || in == "" {
		t.Skip("ERT_GOLDEN / ERT_GOLDEN_IN not set")
	}
	f, err := os.Open(dump)
	if err != nil {
		t.Fatal(err)
	}
	defer f.Close()
	var lines []goldenLine
	sc := bufio.NewScanner(f)
	sc.Buffer(make([]byte, 1<<20), 1<<28)
	for sc.Scan() {
		var l goldenLine
		if err := json.Unmarshal(sc.Bytes(), &l); err != nil {
			t.Fatal(err)
		}
		lines = append(lines, l)
	}
	if len(lines) == 0 || lines[0].Kind != "config" {
		t.Fatal("dump has no config line")
	}
	iq, err := os.ReadFile(in)
	if err != nil {
		t.Fatal(err)
	}

	d := NewDecoder()
	defer d.Close()
	var mu sync.Mutex
	block := 0
	got := map[[3]string]bool{}
	for _, name := range lines[0].Msgtypes {
		d.RegisterProtocol(parityParser{stockConfig(name, lines[0].ChipLen), &mu, &block, got})
	}
	d.Allocate()
	exact := d.Cfg.SymbolLength%8 == 0

	taps := map[int]goldenLine{}
	want := map[[3]string]bool{}
	for _, l := range lines[1:] {
		switch l.Kind {
		case "tap":
			taps[l.Block] = l
		case "cand":
			want[[3]string{itoa(l.Block), l.Preamble, itoa(l.Idx) + ":" + l.Bytes}] = true
		}
	}
	nblocks := len(iq) / d.Cfg.BlockSize2
	for block = 0; block < nblocks; block++ {
		for range d.Decode(iq[block*d.Cfg.BlockSize2 : (block+1)*d.Cfg.BlockSize2]) {
		}
		if tp, ok := taps[block]; ok {
			for which, hexs := range map[int]string{0: tp.Signal, 1: tp.Csum, 2: tp.Quantized, 3: tp.Packed} { // ERTGPU_TAP_*
				ref, _ := hex.DecodeString(hexs)
				if !bytes.Equal(d.Tap(which, int64(block)), ref) {
					t.Errorf("block %d: tap %d differs from the stock decoder", block, which)
				}
			}
		}
	}
	for k := range want {
		if !got[k] {
			t.Errorf("stock candidate missing from the cuda build: %v", k)
		}
	}
	if exact {
		for k := range got {
			if !want[k] {
				t.Errorf("cuda build reports a candidate the stock decoder does not: %v", k)
			}
		}
	}
	t.Logf("%d blocks, %d stock candidates, %d cuda candidates, %d tap blocks", nblocks, len(want), len(got), len(taps))
}
