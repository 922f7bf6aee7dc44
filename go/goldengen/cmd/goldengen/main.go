// goldengen -- runs the STOCK rtlamr decoder and parsers over an IQ file and prints every message as a
// JSON line: the message-level golden vectors (integrity checks, field extraction, r900's own DSP) that
// complement protocol/golden_dump_test.go's decoder-level dump.
//
// Place this directory at <rtlamr>/cmd/goldengen (same module: it imports the stock packages) and run
//
//	go run ./cmd/goldengen -in assets/sample.bin -msgtype scm -symbollength 78 > go_msgs_sample_cl78_scm.jsonl
//
// With -format json or -format xml it writes every message through the encoder rtlamr's -format of that name selects
// (flags.go:147-170) instead: a protocol.LogMessage with Time fixed to 2023-11-14T22:13:20Z and Offset and Length 0, the
// values tests/test_encoders.py hands the C++ encoders for the same messages.
//
// The module needs golang.org/x/xerrors (csv/csv.go:7).  Offline: add
// `replace golang.org/x/xerrors => ./stubs/xerrors` to go.mod and copy stubs/xerrors from this directory
// (an `Errorf` that forwards to fmt.Errorf is all csv.Encode uses).  github.com/bemasher/rtltcp is only
// imported by package main and is not needed here.
//
// flags.go validates -symbollength (flags.go:127-132); the library does not, so 78 (the rate sample.bin
// was captured at) works here.
package main

import (
	"encoding/hex"
	"encoding/json"
	"encoding/xml"
	"flag"
	"fmt"
	"log"
	"os"
	"strings"
	"time"

	"github.com/bemasher/rtlamr/protocol"

	_ "github.com/bemasher/rtlamr/idm"
	_ "github.com/bemasher/rtlamr/netidm"
	_ "github.com/bemasher/rtlamr/r900"
	_ "github.com/bemasher/rtlamr/r900bcd"
	_ "github.com/bemasher/rtlamr/scm"
	_ "github.com/bemasher/rtlamr/scmplus"
)

func main() {
	in := flag.String("in", "", "uint8 IQ file")
	msgtype := flag.String("msgtype", "scm", "comma separated message types")
	chip := flag.Int("symbollength", 72, "the -symbollength flag of rtlamr (really the chip length, main.go:77)")
	format := flag.String("format", "", "json or xml: print each message through rtlamr's encoder instead of the message dump")
	flag.Parse()
	iq, err := os.ReadFile(*in)
	if err != nil {
		log.Fatal(err)
	}
	d := protocol.NewDecoder()
	for _, name := range strings.Split(*msgtype, ",") { // main.go:76-83
		p, err := protocol.NewParser(strings.TrimSpace(name), *chip)
		if err != nil {
			log.Fatal(err)
		}
		d.RegisterProtocol(p)
	}
	d.Allocate() // main.go:86
	if *format != "" {
		encodeAll(&d, iq, *format)
		return
	}
	enc := json.NewEncoder(os.Stdout)
	enc.Encode(map[string]interface{}{"kind": "config", "msgtype": *msgtype, "chip_length": *chip, "cfg": d.Cfg, "input_bytes": len(iq)})
	bs2 := d.Cfg.BlockSize2
	n := 0
	for b := 0; b+1 <= len(iq)/bs2; b++ {
		for msg := range d.Decode(iq[b*bs2 : (b+1)*bs2]) { // main.go:235
			enc.Encode(map[string]interface{}{"kind": "msg", "block": b, "msgtype": msg.MsgType(), "meter_id": msg.MeterID(),
				"meter_type": msg.MeterType(), "checksum": hex.EncodeToString(msg.Checksum()), "record": msg.Record()})
			n++
		}
	}
	enc.Encode(map[string]interface{}{"kind": "end", "blocks": len(iq) / bs2, "messages": n})
}

// newLineEncoder is flags.go's NewLineEncoder: the XML encoder writes no newline after an element.
type newLineEncoder struct{ *xml.Encoder }

func (e newLineEncoder) Encode(v interface{}) error {
	err := e.Encoder.Encode(v)
	fmt.Println()
	return err
}

// encodeAll decodes iq block by block like main.go:235 and encodes each message as main.go:256-266 does.
func encodeAll(d *protocol.Decoder, iq []byte, format string) {
	var enc interface{ Encode(interface{}) error }
	switch format { // flags.go:147-150
	case "json":
		enc = json.NewEncoder(os.Stdout)
	case "xml":
		enc = newLineEncoder{xml.NewEncoder(os.Stdout)}
	default:
		log.Fatalf("-format %q: want json or xml", format)
	}
	t := time.Unix(1700000000, 0).UTC()
	bs2 := d.Cfg.BlockSize2
	for b := 0; b+1 <= len(iq)/bs2; b++ {
		for msg := range d.Decode(iq[b*bs2 : (b+1)*bs2]) {
			if err := enc.Encode(protocol.LogMessage{Time: t, Type: msg.MsgType(), Message: msg}); err != nil {
				log.Fatal(err)
			}
		}
	}
}
